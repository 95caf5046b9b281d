"""The packed states of the fused group-by (csrc/groupby_fused.cu, groupby_dense.cuh, groupby_compact.cuh) and of hash_sum
over group ids, restated on the host, plus an exact group-by reference.

A consume() of the fused group-by takes one of four paths.  Below kPartMinRows rows it is the plain atomic kernel.  From
there the dense path is tried first: a 65,536-row sample sizes a direct-addressed table of packed words
(1 << sb) | (value - vbase), applied in key bands of B2_DENSE_BAND_MB and drained every 2^m rows at most.  When the dense
path declines, the compact path packs each row into one 64-bit tuple (key - kmin) << (vb + 1) | (value - vbase) << 1 | valid
and pre-aggregates it in shared memory, in 32-bit (NARROW) or 64-bit partial sums.  Otherwise the general partitioned path
runs.  Every choice depends only on the data and a few constants, so a test can compute it up front and aim values at the
last bit of a field, at a window's edges, or one step outside.  The constants are read from the sources, so a retune keeps
the cases on target."""
import os
import re
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pyarrow as pa

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arrow_b200", "csrc")
M64 = (1 << 64) - 1


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _find(text, pattern):
    m = re.search(pattern, text)
    assert m, pattern
    return m


def _shift(text, name):
    return 1 << int(_find(text, rf"constexpr [\w ]+ {name} = 1(?:ll|ull)? << (\d+);").group(1))


_FUSED, _DENSE, _COMPACT, _HASHAGG = (_read(n) for n in ("groupby_fused.cu", "groupby_dense.cuh", "groupby_compact.cuh",
                                                         "hash_aggregate.cu"))

K_DENSE_MAX_RANGE = _shift(_DENSE, "kDenseMaxRange")
K_PART_MIN_ROWS = _shift(_FUSED, "kPartMinRows")
K_CHUNK_ROWS = _shift(_FUSED, "kChunkRows")
K_CCHUNK = int(_find(_COMPACT, r"constexpr int kCChunk = (\d+);").group(1))
K_CSLICE_CHUNKS = int(_find(_COMPACT, r"constexpr int kCSliceChunks = (\d+);").group(1))
K_SLICE_TUPLES = K_CCHUNK * K_CSLICE_CHUNKS
K_PRIVATE_MAX_GROUPS = int(_find(_HASHAGG, r"constexpr int kPrivateMaxGroups = (\d+);").group(1))
# the dense path's minimum batch, for the fused table (cn) and by id (n)
DENSE_MIN_ROWS = 1 << int(_find(_FUSED, r"cn < \(1 << (\d+)\)\) return B2_OK;").group(1))
assert DENSE_MIN_ROWS == 1 << int(_find(_FUSED, r"\|\| n < \(1 << (\d+)\) \|\|").group(1))
# rows per slot: n >= ROWS_PER_SLOT * range
ROWS_PER_SLOT = int(_find(_FUSED, r"if \(\(unsigned long long\)cn < (\d+) \* range\) return B2_OK;").group(1))
assert ROWS_PER_SLOT == int(_find(_FUSED, r"\(uint64_t\)n < (\d+) \* num_groups\) return B2_OK;").group(1))
# the padded range may exceed kDenseMaxRange by kDenseMaxRange / RANGE_PAD_DIV
RANGE_PAD_DIV = int(_find(_FUSED, r"if \(range > kDenseMaxRange \+ kDenseMaxRange / (\d+)\) return B2_OK;").group(1))
_m = _find(_FUSED, r"const unsigned long long slack = krange / (\d+) \+ (\d+);")
SLACK_DIV, SLACK_ADD = int(_m.group(1)), int(_m.group(2))
_m = _find(_FUSED, r"const int passes = est <= (\d+) \? 0 : \(est <= (\d+) \? 1 : 2\);")
PASSES_0_MAX, PASSES_1_MAX = int(_m.group(1)), int(_m.group(2))
DEFAULT_BAND_BYTES = int(_find(_FUSED, r"int64_t dense_band_bytes = (\d+)ll << 20;").group(1)) << 20
# m = (M_NUM - vb) / 2, declined below M_MIN; sub-batches at most 2^M_CAP rows
M_NUM = int(_find(_DENSE + _FUSED, r"const int m = \((\d+) - w\.vb\) / 2;").group(1))
M_MIN = int(_find(_FUSED, r"if \(m < (\d+)\) return B2_OK;").group(1))
M_CAP = int(_find(_FUSED, r"const int64_t sub = m >= (\d+) \?").group(1))
SAMPLE_ROWS = int(_find(_FUSED, r"const int64_t step = cn > (\d+) \? cn / \1 : 1;").group(1))
_m = _find(_FUSED, r"const bool narrow = enc\.kb <= (\d+) && enc\.vb <= (\d+);")
NARROW_KB_MAX, NARROW_VB_MAX = int(_m.group(1)), int(_m.group(2))
DENSE_VB_CAP = int(_find(_FUSED, r"value_window\(st, vw, vsigned, (\d+), &w\)\) return B2_OK;\n  DenseBatch").group(1))

INT_TYPES = [pa.int8(), pa.uint8(), pa.int16(), pa.uint16(), pa.int32(), pa.uint32(), pa.int64(), pa.uint64()]


def np_dtype(t: pa.DataType):
    return np.dtype(t.to_pandas_dtype())


def signed(t: pa.DataType) -> bool:
    return pa.types.is_signed_integer(t)


def sample_rows(n: int) -> np.ndarray:
    """rows the 65,536-row sample reads (dense_sample_kernel / compact_value_sample_kernel): 0, step, 2 step, ... < n"""
    step = n // SAMPLE_ROWS if n > SAMPLE_ROWS else 1
    return np.arange(0, n, step, dtype=np.int64)


def enc_keys(keys: np.ndarray) -> np.ndarray:
    """order-preserving uint64 image of the keys: zero-extended bits ^ the sign bit of their width for signed types"""
    w = keys.dtype.itemsize
    u = keys.view(np.dtype(f"u{w}")).astype(np.uint64)
    return u ^ np.uint64(1 << (8 * w - 1)) if keys.dtype.kind == "i" else u


def value_bits(vals: np.ndarray) -> np.ndarray:
    """sign- or zero-extended 64-bit image of the values, as uint64 (what the kernels add)"""
    return vals.astype(np.int64).view(np.uint64) if vals.dtype.kind == "i" else vals.astype(np.uint64)


def bit_width(v: int) -> int:
    return int(v).bit_length()


@dataclass
class Window:
    vb: int
    vbase: int  # mod 2^64: v' = value bits - vbase < 2^vb

    def lo(self, t: pa.DataType) -> int:
        """the smallest value of type t in the window"""
        return _as_type(self.vbase, t)

    def hi(self, t: pa.DataType) -> int:
        return _as_type((self.vbase + (1 << self.vb) - 1) & M64, t)


def _as_type(bits: int, t: pa.DataType) -> int:
    bits &= M64
    return bits - (1 << 64) if signed(t) and bits >> 63 else bits


def value_window(vals: np.ndarray, vvalid: Optional[np.ndarray], rows: np.ndarray, vb_cap: int) -> Optional[Window]:
    """value_window() of groupby_fused.cu over the sampled rows (64-bit values) or the type (narrower ones); None when
    the sampled range does not fit"""
    w = vals.dtype.itemsize
    if w <= 4:
        return Window(8 * w, (-(1 << (8 * w - 1))) & M64 if vals.dtype.kind == "i" else 0)
    if vvalid is not None:
        rows = rows[vvalid[rows]]
    if len(rows) == 0:
        return Window(8, 0)
    flip = 1 << 63 if vals.dtype.kind == "i" else 0
    s = vals[rows].view(np.uint64) ^ np.uint64(flip)
    vmin, vmax = int(s.min()), int(s.max())
    rng = vmax - vmin
    need = bit_width(rng)
    vb = max(8, need + 2)
    vb = min(vb, vb_cap)
    if vb < need or vb < 1 or vb > 62:
        return None
    return Window(vb, ((vmin ^ flip) - (((1 << vb) - 1 - rng) // 2)) & M64)


def _both(a: Optional[np.ndarray], b: Optional[np.ndarray]) -> Optional[np.ndarray]:
    return b if a is None else (a if b is None else a & b)


def in_window(vals: np.ndarray, checked: Optional[np.ndarray], w: Window) -> bool:
    """every value of a `checked` row (valid key and valid value: null-key rows go to the null group unchecked) lies in
    the window"""
    vp = value_bits(vals) - np.uint64(w.vbase)
    bad = vp >> np.uint64(w.vb) != 0
    if checked is not None:
        bad &= checked
    return not bool(bad.any())


@dataclass
class Settings:
    compact: bool = True
    dense: bool = True
    band_bytes: int = DEFAULT_BAND_BYTES

    @staticmethod
    def from_env(env=None):
        env = os.environ if env is None else env
        s = Settings()
        s.compact = not env.get("B2_GROUPBY_COMPACT", "").startswith("0")
        s.dense = not env.get("B2_GROUPBY_DENSE", "").startswith("0")
        bm = env.get("B2_DENSE_BAND_MB", "")
        try:
            if int(bm) > 0:
                s.band_bytes = int(bm) << 20
        except ValueError:
            pass
        return s


@dataclass
class DensePlan:
    """one batch of dense_accumulate: kmin / range index the table ((key bits ^ kflip) - kmin), m / sb size the packed
    fields, `subs` sub-batches of 2^m rows each apply `bands` launches"""
    kmin: int
    kflip: int
    range: int
    window: Window
    m: int
    sb: int
    sub: int
    subs: int
    bands: int
    band_keys: int
    reuse: bool = False

    def launches(self) -> int:
        """kernels dense_accumulate launches: the band launches of every sub-batch, a max-count pass between
        sub-batches and a drain after each"""
        return self.subs * self.bands + (self.subs - 1) + self.subs


@dataclass
class CompactPlan:
    kmin: int
    kb: int
    window: Window
    narrow: bool
    passes: int


@dataclass
class Plan:
    path: str  # dense / compact / general / atomic
    dense: Optional[DensePlan] = None
    compact: Optional[CompactPlan] = None
    why: str = ""  # the first reason a faster path declined


def dense_fields(window: Window, n: int, rng: int, band_bytes: int):
    """(m, sb, sub, subs, bands, band_keys), or None when the window leaves fewer than M_MIN bits for the count"""
    m = (M_NUM - window.vb) // 2
    if m < M_MIN:
        return None
    sub = 1 << min(m, M_CAP)
    band_keys = band_bytes // 8
    return m, window.vb + m, sub, -(-n // sub), -(-rng // band_keys), band_keys


@dataclass
class Held:
    """the dense state a group-by object holds between consumes"""
    kmin: int
    kflip: int
    range: int


@dataclass
class FusedObject:
    """host mirror of one B2GroupBySumCount: what decides the path of its next consume"""
    settings: Settings = field(default_factory=Settings)
    hint: int = 0
    held: Optional[Held] = None
    table_keys: list = field(default_factory=list)  # encoded keys (and None for the null key) that reached the table
    held_keys: list = field(default_factory=list)   # the same for the held dense state

    def _groups(self):
        if not self.table_keys:
            return 0
        ks = [k for k in self.table_keys if k is not None and len(k)]
        n = len(np.unique(np.concatenate(ks))) if ks else 0
        return n + (1 if any(k is None for k in self.table_keys) else 0)

    def plan(self, keys, kvalid, vals, vvalid) -> Plan:
        """the path of consume(keys, vals); kvalid / vvalid are bool arrays (True = valid) or None"""
        n = len(keys)
        if n < K_PART_MIN_ROWS:
            return Plan("atomic")
        vt = vals.dtype
        kflip = (1 << (8 * keys.dtype.itemsize - 1)) if keys.dtype.kind == "i" else 0
        ek = enc_keys(keys)
        rows = sample_rows(n)
        why = ""
        if not self.settings.dense or n < DENSE_MIN_ROWS or vt.kind == "f":
            why = "dense: off, short or float"
        else:
            d = self._try_dense(ek, kvalid, vals, vvalid, rows, n, kflip)
            if isinstance(d, DensePlan):
                return Plan("dense", dense=d)
            why = d
        passes = self._passes()
        if not self.settings.compact or passes == 0 or vt.kind == "f":
            return Plan("general", why=why + "; compact: off, no passes or float")
        kv = ek if kvalid is None else ek[kvalid]
        if len(kv) == 0:
            return Plan("general", why=why + "; compact: every key null")
        kmin, kmax = int(kv.min()), int(kv.max())
        kb = max(1, bit_width(kmax - kmin))
        w = value_window(vals, vvalid, rows, 63 - kb)
        if w is None or kb + w.vb + 1 > 64:
            return Plan("general", why=why + "; compact: fields do not fit")
        if not in_window(vals, _both(kvalid, vvalid), w):
            return Plan("general", why=why + "; compact: a value outside the window")
        narrow = kb <= NARROW_KB_MAX and w.vb <= NARROW_VB_MAX
        return Plan("compact", compact=CompactPlan(kmin, kb, w, narrow, passes), why=why)

    def _passes(self):
        est = self.hint if self.hint > 0 else (self._groups() or (1 << 40))
        return 0 if est <= PASSES_0_MAX else (1 if est <= PASSES_1_MAX else 2)

    def _try_dense(self, ek, kvalid, vals, vvalid, rows, n, kflip):
        sk = ek[rows] if kvalid is None else ek[rows][kvalid[rows]]
        if len(sk) == 0:
            return "dense: no valid key in the sample"
        smin, smax = int(sk.min()), int(sk.max())
        krange = (smax - smin + 1) & M64
        if krange == 0 or krange > K_DENSE_MAX_RANGE:
            return "dense: sampled key range"
        slack = krange // SLACK_DIV + SLACK_ADD
        kmin = smin - slack if smin > slack else 0
        rng = (smax - kmin) + 1 + slack
        h = self.held
        reuse = h is not None and h.kflip == kflip and smin >= h.kmin and smax < ((h.kmin + h.range) & M64)
        if reuse:
            kmin, rng = h.kmin, h.range
        if rng > K_DENSE_MAX_RANGE + K_DENSE_MAX_RANGE // RANGE_PAD_DIV:
            return "dense: padded range"
        if n < ROWS_PER_SLOT * rng:
            return "dense: too few rows per slot"
        w = value_window(vals, vvalid, rows, DENSE_VB_CAP)
        if w is None:
            return "dense: sampled value range"
        f = dense_fields(w, n, rng, self.settings.band_bytes)
        if f is None:
            return "dense: value window too wide"
        idx = (ek - np.uint64(kmin)) if kvalid is None else (ek[kvalid] - np.uint64(kmin))
        if len(idx) and int(idx.max()) >= rng:
            return "dense: a key outside the window"
        if not in_window(vals, _both(kvalid, vvalid), w):
            return "dense: a value outside the window"
        m, sb, sub, subs, bands, band_keys = f
        return DensePlan(kmin, kflip, rng, w, m, sb, sub, subs, bands, band_keys, reuse)

    def consume(self, keys, kvalid, vals, vvalid) -> Plan:
        """plan, then update the mirror as the consume would"""
        p = self.plan(keys, kvalid, vals, vvalid)
        ek = enc_keys(keys)
        if p.path == "dense":
            d = p.dense
            if not d.reuse:
                self._flush()
                self.held = Held(d.kmin, d.kflip, d.range)
                self.held_keys = []
            self.held_keys.append(ek if kvalid is None else ek[kvalid])
            if kvalid is not None and not kvalid.all():
                self.held_keys.append(None)
        else:
            self.table_keys.append(ek if kvalid is None else ek[kvalid])
            if kvalid is not None and not kvalid.all():
                self.table_keys.append(None)
            if p.path != "atomic":
                g = self._groups()
                if self.hint <= 0 or g > self.hint:
                    self.hint = g
        return p

    def _flush(self):
        if self.held is not None:
            self.table_keys.extend(self.held_keys)
            self.held = None


HASHAGG_BAND_BYTES = int(_find(_HASHAGG, r"atoll\(e\) : (\d+)ll\) << 20;").group(1)) << 20
HASHAGG_BAND_MIN_ROWS = 1 << int(_find(_HASHAGG, r"if \(bands < 1 \|\| n < \(1 << (\d+)\)\) bands = 1;").group(1))


@dataclass
class ByIdPlan:
    """one hash_sum consume over group ids: `dense` when dense_sum_count_by_id takes it; otherwise `why`, whether the
    value sample ran, and the dense attempt that a bad row made dense_accumulate decline"""
    dense: Optional[DensePlan]
    why: str = ""
    sampled: bool = False
    attempt: Optional[DensePlan] = None

    def launches(self, vw: int, n: int, num_groups: int) -> int:
        """kernels the consume launches: the value sample (64-bit values), dense_accumulate and the merge on the dense
        path; otherwise whatever ran of those, then the private kernel or the atomic kernel in its L2 bands"""
        if self.dense is not None:
            return (1 if vw == 8 else 0) + self.dense.launches() + 1
        k = (1 if self.sampled and vw == 8 else 0) + (self.attempt.launches() if self.attempt else 0)
        if self.why == "private kernel":
            return k + 1
        band_groups = HASHAGG_BAND_BYTES // 16
        return k + (1 if n < HASHAGG_BAND_MIN_ROWS else max(1, -(-num_groups // band_groups)))


def byid_plan(ids: np.ndarray, num_groups: int, vals: np.ndarray, vvalid: Optional[np.ndarray], skip_nulls=True,
              settings: Optional[Settings] = None) -> ByIdPlan:
    """does hash_sum's consume of (vals, ids) take dense_sum_count_by_id?"""
    settings = settings or Settings()
    n = len(ids)
    has_nulls = vvalid is not None and not vvalid.all()
    if num_groups <= K_PRIVATE_MAX_GROUPS and n >= (1 << 14):
        return ByIdPlan(None, "private kernel")
    if vals.dtype.kind == "f" or not (skip_nulls or not has_nulls):
        return ByIdPlan(None, "float, or has-null flags needed")
    if not settings.dense or n < DENSE_MIN_ROWS or num_groups == 0:
        return ByIdPlan(None, "off or short")
    if num_groups > K_DENSE_MAX_RANGE or n < ROWS_PER_SLOT * num_groups:
        return ByIdPlan(None, "groups")
    w = value_window(vals, vvalid, sample_rows(n), DENSE_VB_CAP)
    if w is None:
        return ByIdPlan(None, "sampled value range", sampled=True)
    f = dense_fields(w, n, num_groups, settings.band_bytes)
    if f is None:
        return ByIdPlan(None, "value window too wide", sampled=True)
    m, sb, sub, subs, bands, band_keys = f
    d = DensePlan(0, 0, num_groups, w, m, sb, sub, subs, bands, band_keys)
    if int(ids.max()) >= num_groups:
        return ByIdPlan(None, "an id out of range", sampled=True, attempt=d)
    if not in_window(vals, vvalid, w):
        return ByIdPlan(None, "a value outside the window", sampled=True, attempt=d)
    return ByIdPlan(d)


# ---- exact reference ----------------------------------------------------------------------------------------------
def _exact_sums(inv: np.ndarray, bits: np.ndarray, groups: int) -> np.ndarray:
    """sum of uint64 `bits` per group id, mod 2^64: four 16-bit limbs summed exactly in float64 (each limb sum stays
    below 2^53 for fewer than 2^37 rows), then recombined with uint64 wrap-around"""
    assert len(bits) < (1 << 37)
    out = np.zeros(groups, dtype=np.uint64)
    for j in range(4):
        limb = ((bits >> np.uint64(16 * j)) & np.uint64(0xFFFF)).astype(np.float64)
        s = np.bincount(inv, weights=limb, minlength=groups)
        out += s.astype(np.uint64) << np.uint64(16 * j)
    return out


def group_sum_count(keys: np.ndarray, kvalid: Optional[np.ndarray], vals: np.ndarray, vvalid: Optional[np.ndarray],
                    key_type: pa.DataType, value_type: pa.DataType) -> pa.Table:
    """hash_sum + hash_count(only_valid) grouped by key: one row per distinct key (ascending) and then the null key if any
    row has one; sums wrap mod 2^64 in int64 (signed values) or uint64; a group whose values are all null has a null sum"""
    n = len(keys)
    kvalid = np.ones(n, bool) if kvalid is None else np.asarray(kvalid, bool)
    vvalid = np.ones(n, bool) if vvalid is None else np.asarray(vvalid, bool)
    ek = enc_keys(keys)[kvalid]
    if len(ek) and int(ek.max()) - int(ek.min()) < (1 << 26):
        base = ek.min()
        off = (ek - base).astype(np.int64)
        present = np.bincount(off) > 0
        uniq_enc = np.nonzero(present)[0].astype(np.uint64) + base
        inv = (np.cumsum(present) - 1)[off]
    else:
        uniq_enc, inv = np.unique(ek, return_inverse=True)
    w = keys.dtype.itemsize
    flip = np.uint64(1 << (8 * w - 1)) if keys.dtype.kind == "i" else np.uint64(0)
    uniq = (uniq_enc ^ flip).astype(np.dtype(f"u{w}")).view(keys.dtype)
    g = len(uniq)
    has_null = not kvalid.all()
    ids = np.empty(n, np.int64)
    ids[kvalid] = inv
    ids[~kvalid] = g
    total = g + (1 if has_null else 0)
    bits = value_bits(vals)
    sel = vvalid
    sums = _exact_sums(ids[sel], bits[sel], total)
    counts = np.bincount(ids[sel], minlength=total).astype(np.int64)
    sum_type = pa.int64() if signed(value_type) else pa.uint64()
    s = sums.view(np.int64) if signed(value_type) else sums
    kmask = np.zeros(total, bool)
    if has_null:
        kmask[g] = True
        uniq = np.concatenate([uniq, np.zeros(1, uniq.dtype)])
    return pa.table({"k": pa.array(uniq, key_type, mask=kmask), "sum": pa.array(s, sum_type, mask=counts == 0),
                     "count": pa.array(counts, pa.int64())})


def sum_by_id(ids: np.ndarray, vals: np.ndarray, vvalid: Optional[np.ndarray], num_groups: int,
              value_type: pa.DataType) -> pa.Array:
    """hash_sum over group ids with skip_nulls and min_count = 1: null where a group has no valid value"""
    vvalid = np.ones(len(ids), bool) if vvalid is None else np.asarray(vvalid, bool)
    ids = ids.astype(np.int64)
    sums = _exact_sums(ids[vvalid], value_bits(vals)[vvalid], num_groups)
    counts = np.bincount(ids[vvalid], minlength=num_groups)
    if signed(value_type):
        return pa.array(sums.view(np.int64), pa.int64(), mask=counts == 0)
    return pa.array(sums, pa.uint64(), mask=counts == 0)


def drain_schedule(ek: np.ndarray, kvalid, vvalid, d: DensePlan) -> list:
    """for each sub-batch but the last: does the max-count guard run the drain after it?  (the count field holds the rows
    with a valid key and a valid value since the last drain; the drain runs when max + rows of the next sub-batch >= 2^m)"""
    n = len(ek)
    ok = _both(kvalid, vvalid)
    idx = (ek - np.uint64(d.kmin)).astype(np.int64)
    acc = np.zeros(d.range, np.int64)
    out = []
    for s in range(d.subs - 1):
        lo, hi = s * d.sub, min(n, (s + 1) * d.sub)
        sel = idx[lo:hi] if ok is None else idx[lo:hi][ok[lo:hi]]
        acc += np.bincount(sel, minlength=d.range)
        nxt = min(d.sub, n - hi)
        drain = int(acc.max()) + nxt >= (1 << d.m)
        if drain:
            acc[:] = 0
        out.append(drain)
    return out


# ---- the cases of test_gpu_groupby_packed_edges.py --------------------------------------------------------------------
@dataclass
class Batch:
    keys: np.ndarray
    kvalid: Optional[np.ndarray]  # True = valid; None = no nulls
    vals: np.ndarray
    vvalid: Optional[np.ndarray]


@dataclass
class Case:
    """batches consumed by one fused group-by; `paths` is the path of each consume, `check(plans, batches)` asserts the
    regime the case is named for"""
    name: str
    key_type: pa.DataType
    value_type: pa.DataType
    make: object  # () -> [Batch]
    paths: list
    env: dict = field(default_factory=dict)
    hint: int = 0
    check: object = None

    def plans(self, batches=None):
        batches = batches if batches is not None else self.make()
        obj = FusedObject(settings=Settings.from_env({**self.env}), hint=self.hint)
        return [obj.consume(b.keys, b.kvalid, b.vals, b.vvalid) for b in batches], batches


def _rng(name):
    return np.random.default_rng(sum(map(ord, name)) * 7919)


def _step(n):
    return n // SAMPLE_ROWS if n > SAMPLE_ROWS else 1


def _unsampled_rows(n, start, count, rng):
    """`count` distinct rows in [start, n) that the sample skips"""
    step = _step(n)
    r = rng.choice(np.arange(start, n), size=count * 2 + 16, replace=False)
    r = r[r % step != 0][:count]
    assert len(r) == count
    return r


def _window_values(rng, n, dtype, lo: int, span: int, vvalid=None):
    """n values of a 64-bit dtype uniform in [lo, lo + span], with lo and lo + span at sampled rows (0 and one step on),
    so the sample sees exactly that range"""
    off = rng.integers(0, span + 1, n, dtype=np.uint64)
    v = (off + np.uint64(lo & M64)).view(dtype) if dtype == np.int64 else off + np.uint64(lo)
    step = _step(n)
    v[0] = np.array(lo & M64, np.uint64).view(dtype) if dtype == np.int64 else lo
    v[step] = np.array((lo + span) & M64, np.uint64).view(dtype) if dtype == np.int64 else lo + span
    if vvalid is not None:
        vvalid[0] = vvalid[step] = True
    return v


def _put(v: np.ndarray, rows, value: int):
    """value (a Python int in the dtype's range, or its bits) into v[rows]"""
    v[rows] = np.array(value & M64, np.uint64).view(np.int64) if v.dtype == np.int64 else \
        (np.uint64(value & M64) if v.dtype == np.uint64 else value)


def _window_of(b: Batch, vb_cap=DENSE_VB_CAP) -> Window:
    return value_window(b.vals, b.vvalid, sample_rows(len(b.keys)), vb_cap)


# ---- dense: value fields full ----
def _dense_hot(vt: pa.DataType, straddle: bool):
    """3 sub-batches of 2^m rows over 1M keys.  hot: sub-batch 0 is one key at the window's top value, sub-batch 1 the same
    key at its bottom value (both fill the count field, the first also the sum field).  straddle: the hot key has
    2^m - 1000 top values at the end of sub-batch 0 and 2000 more at the start of sub-batch 1, so only the drain between
    them keeps its sum inside the field"""
    def make():
        dt = np_dtype(vt)
        m = (M_NUM - 8 * dt.itemsize) // 2
        sub = 1 << m
        n = 3 * sub
        rng = _rng(f"hot{vt}{straddle}")
        keys = rng.integers(0, 1_000_000, n, dtype=np.int32)
        info = np.iinfo(dt)
        vals = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        vvalid = rng.random(n) >= 0.05
        hot = 777_777
        if straddle:
            keys[1000:sub + 2000] = hot
            vals[1000:sub + 2000] = info.max
            vvalid[1000:sub + 2000] = True
        else:
            keys[:2 * sub] = hot
            vals[:sub] = info.max
            vals[sub:2 * sub] = info.min
            vvalid[:2 * sub] = True
        return [Batch(keys, None, vals, vvalid)]

    def check(plans, batches):
        d = plans[0].dense
        assert d.subs == 3 and d.sub == 1 << d.m and d.m == (M_NUM - d.window.vb) // 2
        assert drain_schedule(enc_keys(batches[0].keys), None, batches[0].vvalid, d) == [True, True]

    return Case(f"dense_{'straddle' if straddle else 'hot'}_{vt}", pa.int32(), vt, make, ["dense"], check=check)


def _dense_guard_skips():
    """2 sub-batches, the second shorter than 2^m - (max count): the guard skips the drain, and a hot key with top values in
    both keeps its sum exact"""
    def make():
        m = (M_NUM - 16) // 2
        n = (1 << m) + (1 << 22) + 12345
        rng = _rng("skip")
        keys = rng.integers(-500_000, 500_000, n, dtype=np.int64)
        vals = rng.integers(-32768, 32767, n, dtype=np.int16, endpoint=True)
        hot = np.arange(0, n, 97)
        keys[hot] = 31
        vals[hot] = 32767
        return [Batch(keys, rng.random(n) >= 0.01, vals, rng.random(n) >= 0.1)]

    def check(plans, batches):
        d = plans[0].dense
        b = batches[0]
        assert d.subs == 2 and drain_schedule(enc_keys(b.keys), b.kvalid, b.vvalid, d) == [False]

    return Case("dense_guard_skips_the_drain_int16", pa.int64(), pa.int16(), make, ["dense"], check=check)


def _dense_int8_m27(vt):
    """8-bit values: m = 27.  Sub-batch 0 is 2^27 rows of one key at the top value; a short second sub-batch"""
    def make():
        dt = np_dtype(vt)
        m = (M_NUM - 8) // 2
        n = (1 << m) + (1 << 22)
        rng = _rng(f"m27{vt}")
        keys = np.full(n, 200, np.uint8)
        keys[1 << m:] = rng.integers(0, 256, 1 << 22, dtype=np.uint8)
        info = np.iinfo(dt)
        vals = np.full(n, info.max, dt)
        vals[1 << m:] = rng.integers(info.min, info.max, 1 << 22, dtype=dt, endpoint=True)
        return [Batch(keys, None, vals, None)]

    def check(plans, batches):
        d = plans[0].dense
        assert d.m == 27 and d.subs == 2 and d.sb == 35

    return Case(f"dense_m27_{vt}", pa.uint8(), vt, make, ["dense"], check=check)


# ---- windows of 64-bit values: edges, one step outside ----
_W64 = {  # name -> (value type, lowest sampled value, sampled span)
    "int64_across_0": (pa.int64(), -40_000, 100_000),
    "int64_top": (pa.int64(), (1 << 63) - 1 - 100_000, 100_000),       # the window wraps past INT64_MAX to INT64_MIN
    "int64_bottom": (pa.int64(), -(1 << 63), 100_000),                  # vbase wraps below INT64_MIN
    "uint64_across_2^63": (pa.uint64(), (1 << 63) - 50_000, 100_000),
    "uint64_bottom": (pa.uint64(), 3, 100_000),                          # vbase wraps to the top of uint64
    "uint64_top": (pa.uint64(), (1 << 64) - 1 - 100_000, 100_000),
}


def _edges(name, kind, dense=True):
    """64-bit values whose sample has a 17-bit range (vb = 19: m = 22, the dense limit) or an 18-bit range (vb = 20:
    declined, then compact).  kind: 'on' -- values exactly on both window edges at skipped rows, plus a hot key whose
    sum field fills with top values; 'above' / 'below' -- one value a step outside, at a skipped row"""
    vt, lo, span = _W64[name]
    if not dense:
        span = 200_000  # bit width 18: vb = 20
        lo = lo if lo < (1 << 63) - 300_000 or vt == pa.uint64() else lo - 100_000
        if vt == pa.uint64() and lo > (1 << 64) - 300_000:
            lo -= 100_000

    def make():
        dt = np_dtype(vt)
        n = (1 << 23) + 4099 if dense else (1 << 22) + 4099
        rng = _rng(f"edge{name}{kind}{dense}")
        keys = rng.integers(0, 600_000, n, dtype=np.int64)
        vvalid = rng.random(n) >= 0.05
        vals = _window_values(rng, n, dt, lo, span, vvalid)
        b = Batch(keys, None, vals, vvalid)
        w = _window_of(b)
        rows = _unsampled_rows(n, 2, 64, rng)
        vvalid[rows] = True
        if kind == "on":
            _put(vals, rows[:32], w.lo(vt))
            _put(vals, rows[32:], w.hi(vt))
            # a hot key: every skipped row of sub-batch 0 at the top of the window
            step = _step(n)
            hot = np.arange(1, min(n, 1 << 22))
            hot = hot[hot % step != 0]
            keys[hot] = 4242
            vvalid[hot] = True
            _put(vals, hot, w.hi(vt))
        elif kind == "above":
            _put(vals, rows[:1], (w.vbase + (1 << w.vb)) & M64)
        else:
            _put(vals, rows[:1], (w.vbase - 1) & M64)
        return [b]

    def check(plans, batches):
        w = _window_of(batches[0])
        assert w.vb == (19 if dense else 20), w
        if plans[0].path == "dense":
            assert plans[0].dense.m == M_MIN
        if plans[0].path == "compact":
            assert not plans[0].compact.narrow or w.vb <= NARROW_VB_MAX

    want = ("dense" if dense else "compact") if kind == "on" else "general"
    return Case(f"window_{'vb19' if dense else 'vb20'}_{name}_{kind}", pa.int64(), vt, make, [want], check=check)


# ---- compact fields ----
def _compact(name, kb, need, vt=pa.int64(), hot_top=True, wide_carry=False, key_type=pa.int64()):
    """~3M rows (between kPartMinRows and the dense minimum) whose keys span exactly kb bits and whose sampled values need
    `need` bits; a hot key with 4 slices' worth of rows at the window's top value"""
    def make():
        n = 3_000_000 + 17
        rng = _rng(f"compact{name}")
        kdt = np_dtype(key_type)
        klo = -(1 << (kb - 1)) if kdt.kind == "i" else 0
        keys = rng.integers(0, 300_000, n).astype(np.int64)
        # spread 300k distinct keys over exactly kb bits: key = klo + id * stride, the extremes at rows 0 and 1
        stride = ((1 << kb) - 1) // 299_999
        keys = (keys * stride + klo).astype(kdt)
        keys[0] = klo
        keys[1] = klo + (1 << kb) - 1
        kvalid = rng.random(n) >= 0.01
        kvalid[:2] = True
        dt = np_dtype(vt)
        vvalid = rng.random(n) >= 0.05
        if dt.itemsize == 8:
            span = (1 << (need - 1)) + 12345
            vals = _window_values(rng, n, dt, -(span // 2) if dt.kind == "i" else 1000, span, vvalid)
        else:
            info = np.iinfo(dt)
            vals = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        b = Batch(keys, kvalid, vals, vvalid)
        w = value_window(vals, vvalid, sample_rows(n), 63 - max(1, kb))
        step = _step(n)
        hot = np.arange(100, 100 + 4 * K_SLICE_TUPLES * step // (step - 1) + 64)
        hot = hot[hot % step != 0]
        keys[hot] = keys[1] if not wide_carry else keys[0]
        kvalid[hot] = vvalid[hot] = True
        if hot_top:
            _put(vals, hot, w.hi(vt))
        rows = _unsampled_rows(n, 200_000, 20, rng)
        vvalid[rows] = kvalid[rows] = True
        _put(vals, rows[:10], w.lo(vt))
        _put(vals, rows[10:], w.hi(vt))
        return [b]

    def check(plans, batches):
        c = plans[0].compact
        assert c.kb == kb
        b = batches[0]
        w = value_window(b.vals, b.vvalid, sample_rows(len(b.keys)), 63 - kb)
        assert c.window == w
        if wide_carry:
            assert w.vb > 32 and not c.narrow
        hot = enc_keys(b.keys) == enc_keys(b.keys[1:2] if not wide_carry else b.keys[0:1])[0]
        assert int((hot & b.vvalid & b.kvalid).sum()) >= 2 * K_SLICE_TUPLES

    return Case(f"compact_{name}", key_type, vt, make, ["compact"], check=check)


# ---- bands ----
BAND_MB = 1


def _krange_for(target_range: int) -> int:
    """the sampled key range whose padded range (krange + 2 slack, keys above the slack) is target_range"""
    for kr in range(max(1, target_range - 2 * (target_range // SLACK_DIV) - 2 * SLACK_ADD - 8), target_range + 1):
        if kr + 2 * (kr // SLACK_DIV + SLACK_ADD) == target_range:
            return kr
    return None


def _bands(k: int, delta: int):
    band_keys = (BAND_MB << 20) // 8
    target = k * band_keys + delta

    def make():
        kr = _krange_for(target)
        n = max(DENSE_MIN_ROWS, ROWS_PER_SLOT * target) + 5
        rng = _rng(f"bands{k}{delta}")
        base = 10_000_000
        keys = rng.integers(base, base + kr, n, dtype=np.int64)
        keys[0], keys[_step(n)] = base, base + kr - 1
        kvalid = rng.random(n) >= 0.02
        kvalid[0] = kvalid[_step(n)] = True
        vals = rng.integers(-32768, 32767, n, dtype=np.int16, endpoint=True)
        vvalid = rng.random(n) >= 0.05
        # groups whose every value is null, on each band's first and last slot and the range's last slot
        kmin = base - (kr // SLACK_DIV + SLACK_ADD)
        edge_idx = sorted({i for b in range(1, k + 1) for i in (b * band_keys - 1, b * band_keys)} | {target - 1})
        for idx in edge_idx:
            if base <= kmin + idx < base + kr:
                vvalid[keys == kmin + idx] = False
        return [Batch(keys, kvalid, vals, vvalid)]

    def check(plans, batches):
        d = plans[0].dense
        assert d.range == target and d.bands == -(-target // band_keys) and d.band_keys == band_keys

    return Case(f"bands_{k}x131072{delta:+d}", pa.int64(), pa.int16(), make, ["dense"], env={"B2_DENSE_BAND_MB": str(BAND_MB)},
                check=check)


def _rows_per_slot(inside: bool):
    """n = 4 x range exactly (dense) or one row fewer (declined, then compact)"""
    target = 1_200_000

    def make():
        kr = _krange_for(target)
        n = ROWS_PER_SLOT * target - (0 if inside else 1)
        rng = _rng(f"rps{inside}")
        keys = rng.integers(5_000_000, 5_000_000 + kr, n, dtype=np.int64)
        keys[0], keys[_step(n)] = 5_000_000, 5_000_000 + kr - 1
        vals = rng.integers(0, 255, n, dtype=np.uint8, endpoint=True)
        return [Batch(keys, None, vals, None)]

    def check(plans, batches):
        p = plans[0]
        assert (p.dense.range == target) if inside else ("too few rows per slot" in p.why)

    return Case(f"rows_per_slot_{'inside' if inside else 'outside'}", pa.int64(), pa.uint8(), make,
                ["dense" if inside else "compact"], check=check)


def _max_range_outside():
    """a sampled key range of kDenseMaxRange + 1: declined whatever the rows, then compact"""
    def make():
        n = DENSE_MIN_ROWS + 7
        rng = _rng("maxrange")
        keys = rng.integers(0, K_DENSE_MAX_RANGE + 1, n, dtype=np.int64)
        keys[0], keys[_step(n)] = 0, K_DENSE_MAX_RANGE
        vals = rng.integers(-128, 127, n, dtype=np.int8, endpoint=True)
        return [Batch(keys, None, vals, None)]

    def check(plans, batches):
        assert plans[0].why.startswith("dense: sampled key range")

    return Case("max_range_outside", pa.int64(), pa.int8(), make, ["compact"], check=check)


# ---- keys at their type's ends ----
def _key_ends(kt: pa.DataType, where="both"):
    """keys at the bottom, the top or both ends of their type (8- and 16-bit keys: the whole type)"""
    def make():
        dt = np_dtype(kt)
        info = np.iinfo(dt)
        n = DENSE_MIN_ROWS + 1001
        rng = _rng(f"keyends{kt}")
        span = min(int(info.max) - int(info.min), 200_000)
        half = n // 2
        # half the rows at the bottom of the key type, half at the top (8- and 16-bit keys: the whole type)
        lo = rng.integers(0, span // 2 + 1, half).astype(np.uint64)
        hi = rng.integers(0, span // 2 + 1, n - half).astype(np.uint64)
        if 8 * dt.itemsize <= 16:
            keys = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
            keys[0], keys[1] = info.min, info.max
        else:
            top = np.uint64((1 << (8 * dt.itemsize)) - 1)
            both = np.concatenate([lo, top - hi])
            e = {"both": both, "bottom": np.concatenate([lo, hi]), "top": top - np.concatenate([lo, hi])}[where]
            if where != "top":
                e[0] = 0
            if where != "bottom":
                e[1] = top
            flip = np.uint64(1 << (8 * dt.itemsize - 1)) if dt.kind == "i" else np.uint64(0)
            keys = (e ^ flip).astype(np.dtype(f"u{dt.itemsize}")).view(dt)
        vals = rng.integers(-32768, 32767, n, dtype=np.int16, endpoint=True)
        return [Batch(keys, rng.random(n) >= 0.01, vals, rng.random(n) >= 0.05)]

    # the two ends of a 32-bit type fit one compact tuple, those of a 64-bit type nothing but the general path
    want = "dense" if kt.bit_width <= 16 or where != "both" else ("compact" if kt.bit_width == 32 else "general")
    return Case(f"key_ends_{kt}" + ("" if where == "both" else f"_{where}"), kt, pa.int16(), make, [want])


def _uint64_top_flushed():
    """a dense state over the top of uint64 (the all-ones key included), then a batch with another window: the first state
    is flushed into the hash table, where the all-ones key is the empty marker"""
    def make():
        rng = _rng("u64top")
        n = DENSE_MIN_ROWS + 3
        k1 = (np.uint64(M64) - rng.integers(0, 100_000, n).astype(np.uint64))
        k1[0], k1[_step(n)] = np.uint64(M64), np.uint64(M64 - 99_999)
        k2 = rng.integers(0, 100_000, n).astype(np.uint64)
        v1 = rng.integers(-1000, 1000, n, dtype=np.int32)
        v2 = rng.integers(-1000, 1000, n, dtype=np.int32)
        return [Batch(k1, None, v1.astype(np.int16), rng.random(n) >= 0.05),
                Batch(k2, rng.random(n) >= 0.01, v2.astype(np.int16), None)]

    def check(plans, batches):
        assert not plans[1].dense.reuse

    return Case("uint64_top_then_new_window", pa.uint64(), pa.int16(), make, ["dense", "dense"], check=check)


def _held_window(outside: bool):
    """a second batch whose sample lies inside the held window: reused (dense), or -- with one key just outside the held
    range at a skipped row -- declined without touching the held state"""
    def make():
        rng = _rng(f"held{outside}")
        n = DENSE_MIN_ROWS + 11
        k1 = rng.integers(-300_000, 300_000, n, dtype=np.int64)
        k1[0], k1[_step(n)] = -300_000, 299_999
        k2 = rng.integers(-200_000, 200_000, n, dtype=np.int64)
        b1 = Batch(k1, rng.random(n) >= 0.01, rng.integers(-128, 127, n, dtype=np.int8, endpoint=True), None)
        b2 = Batch(k2, None, rng.integers(-128, 127, n, dtype=np.int8, endpoint=True), rng.random(n) >= 0.1)
        if outside:
            obj = FusedObject()
            d = obj.consume(b1.keys, b1.kvalid, b1.vals, b1.vvalid).dense
            row = _unsampled_rows(n, 1000, 1, rng)[0]
            k2[row] = d.kmin + d.range - (1 << 63)  # the first encoded key past the held range (signed: flip the sign bit)
        return [b1, b2]

    def check(plans, batches):
        if not outside:
            assert plans[1].dense.reuse
        else:
            assert "key outside" in plans[1].why

    return Case(f"held_window_{'one_key_outside' if outside else 'reused'}", pa.int64(), pa.int8(), make,
                ["dense", "compact" if outside else "dense"], check=check)


def fused_cases():
    cs = []
    for vt in (pa.int16(), pa.uint16()):
        cs += [_dense_hot(vt, False), _dense_hot(vt, True)]
    cs.append(_dense_guard_skips())
    cs += [_dense_int8_m27(pa.int8()), _dense_int8_m27(pa.uint8())]
    for name in _W64:
        for kind in ("on", "above", "below"):
            cs.append(_edges(name, kind))
    for name in ("int64_across_0", "uint64_top"):
        for kind in ("on", "above"):
            cs.append(_edges(name, kind, dense=False))
    cs += [
        _compact("kb40_vb23_full", 40, 21),
        _compact("kb42_vb_cut_to_21", 42, 20),
        _compact("kb31_vb19_narrow", 31, 17),
        _compact("kb31_vb20_wide", 31, 18),
        _compact("kb32_vb19_wide", 32, 17),
        _compact("kb23_vb40_wide_carry", 23, 38, wide_carry=True),
        _compact("kb31_int32_values_full", 31, 0, vt=pa.int32(), key_type=pa.int32()),
        _compact("kb17_uint32_values", 17, 0, vt=pa.uint32(), key_type=pa.uint32()),
    ]
    for delta in (-1, 0, 1):
        cs.append(_bands(3, delta))
    cs += [_rows_per_slot(True), _rows_per_slot(False), _max_range_outside()]
    for kt in INT_TYPES:
        cs.append(_key_ends(kt))
        if kt.bit_width >= 32:
            cs += [_key_ends(kt, "bottom"), _key_ends(kt, "top")]
    cs += [_uint64_top_flushed(), _held_window(False), _held_window(True)]
    return cs


# ---- hash_sum over group ids ----
@dataclass
class ByIdCase:
    """consumes of one hash_sum aggregator: each (ids, vals, vvalid, offset) is consumed from row `offset` of device copies
    of the arrays; `dense` is whether each consume takes dense_sum_count_by_id"""
    name: str
    value_type: pa.DataType
    num_groups: int
    make: object  # () -> [(ids, vals, vvalid, offset)]
    dense: list
    env: dict = field(default_factory=dict)
    check: object = None

    def plans(self, consumes=None):
        consumes = consumes if consumes is not None else self.make()
        st = Settings.from_env(self.env)
        return [byid_plan(i[o:], self.num_groups, v[o:], None if vv is None else vv[o:], settings=st)
                for i, v, vv, o in consumes], consumes


def _byid_from(case: Case, num_groups: int):
    """a fused case's batch with its keys mapped onto group ids in [0, num_groups), the largest id used"""
    def make():
        b = case.make()[0]
        k = enc_keys(b.keys)
        ids = ((k - k.min()) % np.uint64(num_groups)).astype(np.uint32)
        ids[-1] = num_groups - 1
        return [(ids, b.vals, b.vvalid, 0)]
    return make


def _byid_offsets(vt: pa.DataType):
    """three consumes from odd offsets of one pair of sliced arrays, each >= the dense minimum, adding into one state in
    bands of 1 MB"""
    groups = 500_000

    def make():
        rng = _rng(f"byidoff{vt}")
        dt = np_dtype(vt)
        n = 3 * DENSE_MIN_ROWS + 100
        ids = rng.integers(0, groups, n, dtype=np.uint32)
        ids[::1001] = groups - 1
        if dt.itemsize == 8:
            vals = _window_values(rng, n, dt, -60_000 if dt.kind == "i" else (1 << 63) - 60_000, 100_000)
        else:
            info = np.iinfo(dt)
            vals = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        vvalid = rng.random(n) >= 0.1
        cuts = [1, DENSE_MIN_ROWS + 5, 2 * DENSE_MIN_ROWS + 40]
        return [(ids[:cuts[1]], vals[:cuts[1]], vvalid[:cuts[1]], 1),
                (ids[:cuts[2]], vals[:cuts[2]], vvalid[:cuts[2]], cuts[1]),
                (ids, vals, vvalid, cuts[2])]

    return ByIdCase(f"byid_offsets_bands_{vt}", vt, groups, make, [True, True, True], env={"B2_DENSE_BAND_MB": "1"})


def _byid_groups(num_groups: int, rows: int, want: bool, tag: str):
    def make():
        rng = _rng(f"byidg{tag}")
        ids = rng.integers(0, num_groups, rows, dtype=np.uint32)
        ids[-1] = num_groups - 1
        return [(ids, rng.integers(-128, 127, rows, dtype=np.int8, endpoint=True), None, 0)]
    return ByIdCase(f"byid_{tag}", pa.int8(), num_groups, make, [want])


def byid_cases():
    cs = []
    for vt in (pa.int16(), pa.uint16()):
        for straddle in (False, True):
            c = _dense_hot(vt, straddle)
            cs.append(ByIdCase("byid_" + c.name, vt, 1_000_000, _byid_from(c, 1_000_000), [True]))
    for name, kind in (("int64_across_0", "on"), ("int64_top", "on"), ("uint64_bottom", "on"), ("uint64_across_2^63", "on"),
                       ("int64_across_0", "above"), ("uint64_bottom", "below")):
        c = _edges(name, kind)
        cs.append(ByIdCase("byid_" + c.name, c.value_type, 600_000, _byid_from(c, 600_000), [kind == "on"]))
    c = _edges("int64_across_0", "on", dense=False)
    cs.append(ByIdCase("byid_" + c.name, c.value_type, 600_000, _byid_from(c, 600_000), [False]))
    for vt in (pa.int8(), pa.uint16(), pa.int64()):
        cs.append(_byid_offsets(vt))
    cs += [_byid_groups(K_DENSE_MAX_RANGE, ROWS_PER_SLOT * K_DENSE_MAX_RANGE, True, "max_groups"),
           _byid_groups(K_DENSE_MAX_RANGE + 1, ROWS_PER_SLOT * K_DENSE_MAX_RANGE + 4, False, "max_groups_plus_1"),
           _byid_groups(1_200_000, ROWS_PER_SLOT * 1_200_000, True, "rows_per_group_inside"),
           _byid_groups(1_200_000, ROWS_PER_SLOT * 1_200_000 - 1, False, "rows_per_group_outside")]
    return cs
