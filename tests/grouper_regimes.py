"""A host restatement of grouper_run's choices (csrc/grouper.cu) for one fixed-width key column, and the case table the
GPU edge tests run.

HostGrouper is two things at once:
  * the exact reference: ids in first-occurrence order, uniques, Lookup (unknown -> null), by raw key bits;
  * a model of the device's regime per Consume: direct or hash mode, the direct window (lo, cap), the hash table's
    capacity before and after, the insert-overflow regrows, the rehash overflows inside grouper_rebuild, the
    load-factor rebuild, and whether new groups are flagged by slots (cap <= n) or by rows.
The table is simulated by sequential linear probing of the distinct keys in first-occurrence order.  The device probes in
parallel, so a neighbourhood that is nearly full may overflow in one and not the other; the cases below keep their
clusters well past kMaxProbe (or well below it) so both agree."""
import numpy as np
import pyarrow as pa

from oracle import arrow_oracle as ora
from tests import hash_keys as hk

SIGN_FLIP = {pa.int8(): 1 << 7, pa.int16(): 1 << 15, pa.int32(): 1 << 31, pa.int64(): 1 << 63}


def key_bits(arr: pa.Array):
    """(zero-extended raw key bits as uint64, validity) of a fixed-width array"""
    v = ora.values(arr)
    u = v.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[v.dtype.itemsize]).astype(np.uint64)
    return u, ora.validity(arr)


def same_bits(a: pa.Array, b: pa.Array) -> bool:
    """equal type, length, validity and raw bits at the valid slots (NaN payloads and -0.0 included)"""
    if a.type != b.type or len(a) != len(b):
        return False
    (ab, av), (bb, bv) = key_bits(a), key_bits(b)
    return bool(np.array_equal(av, bv) and np.array_equal(ab[av], bb[bv]))


class HostGrouper:
    def __init__(self, key_type: pa.DataType, direct_enabled: bool = True):
        self.type = key_type
        self.flip = SIGN_FLIP.get(key_type, 0)
        self.direct_eligible = direct_enabled and pa.types.is_integer(key_type)
        self.direct = False
        self.lo = self.dcap = 0
        self.obs_min, self.obs_max = hk.M64, 0
        self.cap = 0
        self.slots = {}      # simulated hash table: slot -> key bits
        self.ids = {}        # key bits (None = null) -> id
        self.uniques = []    # key bits (None = null) in id order
        self.log = []        # one outcome dict per Consume

    # ---- the simulated hash table --------------------------------------------------------------------------------
    def _insert(self, key):
        if key is None or key == hk.EMPTY_KEY:
            return True       # the two extra slots
        s = hk.fmix64(key) & (self.cap - 1)
        for _ in range(hk.MAX_PROBE):
            cur = self.slots.get(s)
            if cur is None:
                self.slots[s] = key
                return True
            if cur == key:
                return True
            s = (s + 1) & (self.cap - 1)
        return False

    def _rebuild(self, cap, out):
        while True:
            self.cap, self.slots = cap, {}
            if all(self._insert(k) for k in self.uniques):
                return
            out["rehash_overflows"] += 1
            cap *= 4

    # ---- Consume / Lookup ------------------------------------------------------------------------------------------
    def consume(self, arr: pa.Array) -> np.ndarray:
        bits, valid = key_bits(arr)
        n = len(arr)
        out = dict(n=n, mode=None, lo=None, dcap=None, cap_before=self.cap, cap_after=self.cap, regrows=0,
                   rehash_overflows=0, load_rebuild=False, flag=None, fallback=False, reseat=None, clamped=False)
        self.log.append(out)
        # first occurrences of this batch, in row order
        new_keys = []
        if n:
            u, first = np.unique(bits[valid], return_index=True)
            rows = np.flatnonzero(valid)[first]
            cand = sorted(zip(rows.tolist(), u.tolist()))
            if (~valid).any():
                cand = sorted(cand + [(int(np.flatnonzero(~valid)[0]), None)])
            new_keys = [k for _, k in cand if k not in self.ids]
        if n == 0:
            return np.zeros(0, np.uint32)
        if self.direct_eligible:
            ords = (bits[valid] ^ np.uint64(self.flip)) if valid.any() else None
            if ords is not None:
                self.obs_min = min(self.obs_min, int(ords.min()))
                self.obs_max = max(self.obs_max, int(ords.max()))
            seen = self.obs_min <= self.obs_max
            lo_need, hi_need = (self.obs_min, self.obs_max) if seen else (0, 0)
            width = hi_need - lo_need
            roomy = max(n * hk.ROOMY_MUL, hk.ROOMY_MIN)
            if width < hk.DIRECT_MAX_RANGE and (self.direct or width < roomy):
                if not self.direct or lo_need < self.lo or hi_need - self.lo >= self.dcap:
                    if self.direct:
                        out["reseat"] = "below" if lo_need < self.lo else "above"
                    self._build_direct(lo_need, hi_need, out)
            else:
                was = self.direct
                self.direct = self.direct_eligible = False
                if was:
                    out["fallback"] = True
                    self._rebuild(hk.next_pow2(len(self.uniques) * 4 + 1024), out)
        if self.direct:
            out.update(mode="direct", lo=self.lo, dcap=self.dcap)
        else:
            out["mode"] = "hash"
            if self.cap == 0:
                n_ = n
                guess = hk.GUESS_FLOOR if n_ < hk.GUESS_SMALL else (
                    hk.GUESS_MUL * n_ if n_ < (1 << hk.GUESS_MID) else 1 << hk.GUESS_TOP)
                self._rebuild(hk.next_pow2(guess), out)
                out["cap_before"] = self.cap
            while not all(self._insert(k) for k in new_keys):
                out["regrows"] += 1
                self._rebuild(self.cap * 4, out)
            out["flag"] = "slots" if self.cap <= n else "rows"
        for k in new_keys:
            self.ids[k] = len(self.uniques)
            self.uniques.append(k)
        if not self.direct and len(self.uniques) * 2 > self.cap:
            out["load_rebuild"] = True
            self._rebuild(hk.next_pow2(len(self.uniques) * 4), out)
        out["cap_after"] = self.cap
        return self._ids_of(bits, valid)[0]

    def _build_direct(self, mn, mx, out):
        span = mx - mn + 1
        cap = min(hk.next_pow2(max(span * 2, hk.DIRECT_FLOOR)), hk.DIRECT_MAX_RANGE)
        pad = (cap - span) // 2
        lo = mn - pad if mn >= pad else 0
        if lo > hk.M64 - (cap - 1):
            lo = hk.M64 - (cap - 1)
            out["clamped"] = True
        self.lo, self.dcap, self.direct = lo, cap, True

    def _ids_of(self, bits, valid):
        ids = np.zeros(len(bits), np.uint32)
        ok = np.zeros(len(bits), bool)
        if valid.any():
            u, inv = np.unique(bits[valid], return_inverse=True)
            got = np.array([self.ids.get(k, -1) for k in u.tolist()], np.int64)
            g = got[inv]
            ids[valid] = np.where(g >= 0, g, 0)
            ok[valid] = g >= 0
        if (~valid).any() and None in self.ids:
            ids[~valid] = self.ids[None]
            ok[~valid] = True
        return ids, ok

    def lookup(self, arr: pa.Array) -> pa.Array:
        ids, ok = self._ids_of(*key_bits(arr))
        return ora.make_array(pa.uint32(), ids, ok)

    def get_uniques(self) -> pa.Array:
        valid = np.array([k is not None for k in self.uniques], bool)
        bits = np.array([0 if k is None else k for k in self.uniques], np.uint64)
        dt = ora.np_dtype(self.type)
        vals = bits.astype({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(dt).itemsize]).view(dt)
        return ora.make_array(self.type, vals, valid)


# ---- the case table -------------------------------------------------------------------------------------------------
EMPTY_I64 = np.int64(-1)


def _arr(vals, t, nulls=None):
    """an 8-byte key column from raw 64-bit words"""
    return pa.array(np.ascontiguousarray(vals).view(ora.np_dtype(t)), t, mask=nulls)


def _spread(keys, n, seed):
    """n rows over `keys`: every key at least once, first occurrences shuffled, duplicates spread through the batch"""
    rng = np.random.default_rng(seed)
    rows = np.concatenate([keys, rng.choice(keys, n - len(keys))])
    rng.shuffle(rows)
    return rows


def cluster(n, bits, seed, dtype=np.int64):
    """n distinct keys whose hash64 shares its low `bits` bits: one home slot in every table of up to 2^bits slots"""
    return hk.keys_with_fields(n, hk.slot_field(bits), seed, dtype)


def narrow_cases():
    """name -> (key type, B2_GROUPER_DIRECT enabled, [batches]).  Clustered keys are 300 distinct keys sharing their low
    bits, so a neighbourhood needs more than kMaxProbe = 256 probes until the table outgrows the shared bits."""
    i64, f64, u64 = pa.int64(), pa.float64(), pa.uint64()
    c16 = cluster(300, 16, 1)
    fill = hk.filler_keys(12000, [hk.slot_field(16)], 2)
    c24 = cluster(300, 24, 3)
    fill24 = hk.filler_keys(10000, [hk.slot_field(24)], 4)
    rng = np.random.default_rng(5)
    big = np.concatenate([c24, rng.choice(np.concatenate([c24, fill24]), (1 << hk.GUESS_MID) + 5 - 300)])
    rng.shuffle(big)
    special = np.concatenate([c16[:280], [EMPTY_I64]])
    n_sp = len(special) + 200
    sp_rows = _spread(special, n_sp, 6)
    sp_nulls = np.zeros(n_sp, bool)
    sp_nulls[rng.choice(n_sp, 20, replace=False)] = True
    dense = hk.consecutive_keys_with_low_bits(300, 14)
    cases = {
        # first batch below GUESS_SMALL rows: 1024 -> 4096 -> 16384 -> 65536 all overflow
        "first_small": (i64, True, [_arr(_spread(c16, hk.GUESS_SMALL - 1, 7), i64)]),
        # first batch of >= 2^22 rows: the 2^23 first guess overflows on keys that share 24 bits
        "first_large": (i64, True, [_arr(big, i64)]),
        # the clustered keys arrive after thousands of groups exist
        "later_batch": (i64, True, [_arr(fill[:5000], i64),
                                    _arr(_spread(np.concatenate([c16, fill[:3000]]), 8000, 8), i64)]),
        # float64 keys with the all-ones bit pattern (a NaN) and nulls mixed into a clustered batch
        "special_in_cluster": (f64, True, [_arr(sp_rows, f64, sp_nulls)]),
        # a small first table, then a batch at least as long as it: new groups flagged by slots, incl. the two extras
        "flag_slots_special": (i64, True, [
            _arr(fill[:100], i64),
            _arr(np.concatenate([[EMPTY_I64], np.tile(fill[:100], 20), fill[5000:5300], [0]]), i64,
                 np.concatenate([np.zeros(2301, bool), [True]]))]),
        # the special keys as the only row, the first row and the last row, new groups flagged by rows
        "flag_rows_special": (u64, False, [
            _arr(np.array([hk.EMPTY_KEY], np.uint64), u64),
            pa.array([None], u64),
            _arr(np.concatenate([fill[6000:6100].view(np.uint64), [np.uint64(hk.EMPTY_KEY)]]), u64),
            _arr(np.concatenate([[np.uint64(0)], c16.view(np.uint64), fill[6100:6200].view(np.uint64)]), u64,
                 np.concatenate([[True], np.zeros(400, bool)]))]),
        # both special keys NEW as the first and the last row of a batch whose new groups are flagged by rows
        "flag_rows_special_ends": (u64, False, [
            _arr(np.concatenate([[np.uint64(0)], fill[6200:6300].view(np.uint64), [np.uint64(hk.EMPTY_KEY)]]), u64,
                 np.concatenate([[True], np.zeros(101, bool)])),
            _arr(np.concatenate([[np.uint64(hk.EMPTY_KEY)], c16.view(np.uint64), [np.uint64(0)]]), u64,
                 np.concatenate([np.zeros(301, bool), [True]]))]),
        # load above 1/2 after a later batch: rebuilt at next_pow2(4 * groups)
        "load_rebuild": (f64, True, [_arr(fill[7000:7400], f64), _arr(fill[7400:7700], f64)]),
        # uniques stored in direct mode collide at the capacity the direct -> hash fallback picks: grouper_rebuild's
        # rehash overflows twice (4096, 16384) before 65536 fits.  The wide batch holds none of them, so no insert
        # overflow rebuilds the table again and only the rehash loop can have put every stored key back
        "fallback_rehash": (i64, True, [_arr(_spread(dense, 700_000, 9), i64),
                                        _arr(np.concatenate([[1 << 40], fill[8000:8100]]), i64)]),
    }
    return cases


def _log2(v):
    assert v & (v - 1) == 0
    return v.bit_length() - 1


def fused_atomic_keys():
    """(clustered, second, filler) int64 keys for the fused group-by's atomic path: kMaxProbe + 44 keys on one home
    slot in every table up to 16x its first size, so the grow-and-retry-pending loop runs several rounds"""
    bits = _log2(hk.FUSED_FIRST_CAP) + 4
    c = cluster(hk.MAX_PROBE + 44, bits, 31)
    fill = hk.filler_keys(3000, [hk.slot_field(bits)], 32, exclude=c)
    return c, fill[:10], fill


def fused_partitioned_keys():
    """(clustered, pre-slot, filler) int64 keys for the partitioned path.  clustered: kMaxProbe + 44 keys on one home
    slot in the first table (FUSED_PART_CAP) and the next one, hence also in one digit of both radix passes.  pre-slot:
    2 * kPreProbe + 4 keys with equal radix digits and one pre-aggregation slot: more distinct keys in one slot of a
    slice than kPreProbe probes can reach"""
    digit_bits = 2 * _log2(hk.PART_RADIX)
    bits = _log2(hk.FUSED_PART_CAP) + 1
    assert bits >= digit_bits
    c = cluster(hk.MAX_PROBE + 44, bits, 41)
    pre_fields = [(0, digit_bits, 0x1357)] + hk.pre_slot_field()
    pre = hk.keys_with_fields(2 * hk.PRE_PROBE + 4, pre_fields, 42)
    fill = hk.filler_keys(3000, [hk.slot_field(bits), pre_fields], 43, exclude=np.concatenate([c, pre]))
    return c, pre, fill


def fused_atomic_grows(keys):
    """rounds of the atomic path's grow-and-retry loop the clustered keys force: the table grows to
    max(4 * groups, 2 * cap) while more than kMaxProbe of them share a home slot"""
    h = hk.fmix64_np(keys.view(np.uint64))
    cap, rounds = hk.FUSED_FIRST_CAP, 0
    while np.bincount((h & np.uint64(cap - 1)).astype(np.int64)).max() > hk.MAX_PROBE:
        cap = hk.next_pow2(max(4 * len(keys), 2 * cap))
        rounds += 1
    return rounds


def _window(t, lo_val, width, n, seed, nulls=0.0):
    """n values of type t in [lo_val, lo_val + width], both ends present"""
    rng = np.random.default_rng(seed)
    v = [lo_val + int(x) for x in rng.integers(0, width + 1, n)]
    v[0], v[-1] = lo_val, lo_val + width
    mask = rng.random(n) < nulls if nulls else None
    if mask is not None:
        mask[0] = mask[-1] = False
    return pa.array(np.array(v, dtype=ora.np_dtype(t)), t, mask=mask)


def direct_cases():
    """name -> (key type, [batches]): the direct-addressed window's edges"""
    i8, i16, i32, i64, u64 = pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint64()
    cases = {}
    for n in (4000, 10000):   # both sides of ROOMY_MIN / ROOMY_MUL
        roomy = max(n * hk.ROOMY_MUL, hk.ROOMY_MIN)
        cases[f"roomy_n{n}_below"] = (i32, [_window(i32, -1000, roomy - 1, n, n)])
        cases[f"roomy_n{n}_at"] = (i32, [_window(i32, -1000, roomy, n, n + 1)])
    cases["widen_to_limit"] = (i64, [_window(i64, 5, 1000, 2000, 1),
                                     _window(i64, 5, hk.DIRECT_MAX_RANGE - 1, 3000, 2),
                                     _window(i64, 5, hk.DIRECT_MAX_RANGE, 3000, 3)])
    cases["reseat_below_above"] = (i32, [_window(i32, 100_000, 100, 3000, 4, 0.05),
                                         _window(i32, 50_000, 100, 3000, 5),
                                         _window(i32, 400_000, 100, 3000, 6, 0.05)])
    cases["int8_full"] = (i8, [_window(i8, -128, 255, 2000, 7, 0.1), _window(i8, -5, 10, 100, 8)])
    cases["int16_ends"] = (i16, [_window(i16, -32768, 100, 2000, 9), _window(i16, 32767 - 100, 100, 2000, 10),
                                 _window(i16, -300, 600, 2000, 11, 0.1)])
    cases["int32_ends"] = (i32, [_window(i32, -2**31, 1000, 3000, 12), _window(i32, -500, 1000, 3000, 13),
                                 _window(i32, 2**31 - 1001, 1000, 3000, 14)])
    cases["int64_ends"] = (i64, [_window(i64, 2**63 - 1001, 1000, 3000, 15, 0.02), _window(i64, -700, 1400, 3000, 16)])
    cases["int64_min"] = (i64, [_window(i64, -2**63, 1000, 3000, 17)])
    cases["uint64_top"] = (u64, [_window(u64, 2**64 - 300, 299, 2000, 18, 0.05), _window(u64, 2**64 - 2000, 1000, 2000, 19)])
    cases["all_null_first"] = (i32, [pa.array([None] * 50, i32), _window(i32, 70_000, 500, 2000, 20)])
    return cases


def expected_outcomes():
    """(case, batch, key, value) facts the case tables are built to reach; the CPU test checks them against the model"""
    return [
        ("first_small", 0, "regrows", 4), ("first_small", 0, "cap_before", hk.GUESS_FLOOR), ("first_small", 0, "flag", "rows"),
        ("first_large", 0, "cap_before", 1 << hk.GUESS_TOP), ("first_large", 0, "regrows", 1), ("first_large", 0, "flag", "rows"),
        ("later_batch", 1, "regrows", 2),
        ("special_in_cluster", 0, "regrows", 4),
        ("flag_slots_special", 1, "flag", "slots"),
        ("flag_rows_special", 0, "flag", "rows"), ("flag_rows_special", 1, "flag", "rows"),
        ("flag_rows_special", 3, "regrows", 4),
        ("flag_rows_special_ends", 0, "flag", "rows"), ("flag_rows_special_ends", 1, "flag", "rows"),
        ("flag_rows_special_ends", 1, "regrows", 4),
        ("load_rebuild", 1, "load_rebuild", True),
        ("fallback_rehash", 0, "mode", "direct"), ("fallback_rehash", 1, "fallback", True),
        ("fallback_rehash", 1, "rehash_overflows", 2),
        ("roomy_n4000_below", 0, "mode", "direct"), ("roomy_n4000_at", 0, "mode", "hash"),
        ("roomy_n10000_below", 0, "mode", "direct"), ("roomy_n10000_at", 0, "mode", "hash"),
        ("widen_to_limit", 1, "mode", "direct"), ("widen_to_limit", 1, "dcap", hk.DIRECT_MAX_RANGE),
        ("widen_to_limit", 2, "fallback", True),
        ("reseat_below_above", 1, "reseat", "below"), ("reseat_below_above", 2, "reseat", "above"),
        ("uint64_top", 0, "clamped", True), ("all_null_first", 0, "mode", "direct"),
        ("int64_ends", 1, "fallback", True), ("int64_min", 0, "mode", "direct"),
    ]


def run_model(cases_with_flag):
    """case name -> the HostGrouper after consuming every batch"""
    out = {}
    for name, (t, direct_on, batches) in cases_with_flag.items():
        g = HostGrouper(t, direct_on)
        for b in batches:
            g.consume(b)
        out[name] = g
    return out
