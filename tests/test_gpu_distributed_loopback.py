"""The multi-GPU group-by and sort (arrow_b200.distributed over DeviceOps) with P ranks in one process on one GPU, against
exact references.

NCCL refuses two ranks on one device, so here every rank is a thread with a Context and a DeviceOps of its own, and the
ranks exchange through LoopbackExchange, an in-process implementation of the transport interface.  Everything between the
kernels runs as it does on P GPUs: splitting off the null-key group, the hash owner rule, the partition plan, the
sample and splitters, the metadata row, the merge of the partials and the unsigned <-> signed tensor views.

Inputs are split into uneven row-range shards, some of them empty.  Group-by results are compared per key, keyed by the
key's bits: counts exactly, integer sums wrapped to 64 bits exactly, float sums within the bound of any summation order
around math.fsum.  Sorts are compared with sort_ref.sort_indices_np."""
import math
import threading

import numpy as np
import pyarrow as pa
import pytest
import torch

from tests import exact_ref as er
from tests import sort_ref
from tests.hash_keys import fmix64_np
from tests.util import SEED

pytestmark = pytest.mark.gpu

WORLDS = (2, 3, 4, 8)
MAX_RANKS = max(WORLDS)
BARRIER_TIMEOUT = 300.0   # seconds; a failing rank breaks the barrier at once, so this bounds only a rank that never arrives


# ---------------------------------------------------------------------------------------------------------------------
# P ranks on threads
# ---------------------------------------------------------------------------------------------------------------------
class _Hub:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=BARRIER_TIMEOUT)
        self.slots = [None] * world


class LoopbackExchange:
    """The transport interface of arrow_b200.distributed (as TorchExchange / B2CommExchange) between the threads of one
    process.  A collective publishes host copies (.cpu() waits for the sender's stream), waits for every rank to publish,
    copies what it receives back to the device on its own stream, then waits for every rank to finish reading, so no rank
    overwrites its slot while a peer still reads it.  Correct, not fast."""

    def __init__(self, hub, rank):
        self.hub, self.world, self.rank, self.stats = hub, hub.world, rank, {}

    def _collective(self, mine, read):
        hub = self.hub
        hub.slots[self.rank] = mine
        hub.barrier.wait()
        out = read(hub.slots)
        hub.barrier.wait()
        return out

    def _all_gather(self, t):
        return self._collective(t.cpu(), lambda slots: torch.stack(slots).to(t.device))

    def all_gather_i64(self, row):
        assert row.dtype == torch.int64
        return self._all_gather(row)

    def all_gather_bytes(self, buf):
        assert buf.dtype == torch.uint8
        return self._all_gather(buf)

    def all_to_all_columns(self, columns, send_rows, recv_rows):
        assert len(send_rows) == self.world and len(recv_rows) == self.world, (send_rows, recv_rows)
        bounds = np.cumsum([0] + [int(x) for x in send_rows])
        host = [c.cpu() for c in columns]
        assert all(len(h) == bounds[-1] for h in host), "columns and send counts disagree"
        mine = [[h[bounds[d]: bounds[d + 1]] for h in host] for d in range(self.world)]

        def read(slots):
            parts = [slots[src][self.rank] for src in range(self.world)]
            assert [len(p[0]) for p in parts] == [int(x) for x in recv_rows], "receive counts disagree with what was sent"
            return [torch.cat([p[i] for p in parts]).to(c.device) for i, c in enumerate(columns)]

        outs = self._collective(mine, read)
        self.stats = {"alltoall_bytes": sum(c.element_size() * (int(bounds[-1]) - int(send_rows[self.rank])) for c in columns)}
        return outs


def run_ranks(world, fn):
    """fn(rank, exchange) on `world` threads, one per rank; the results in rank order, or the first rank's own error (a
    rank that fails breaks the barrier, so its peers fail too, with BrokenBarrierError)"""
    hub = _Hub(world)
    results, errors = [None] * world, [None] * world

    def body(rank):
        try:
            results[rank] = fn(rank, LoopbackExchange(hub, rank))
        except BaseException as e:
            errors[rank] = e
            hub.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,), name=f"loopback-rank-{r}") for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    raised = [e for e in errors if e is not None]
    if raised:
        raise next((e for e in raised if not isinstance(e, threading.BrokenBarrierError)), raised[0])
    return results


@pytest.fixture(scope="module")
def rank_ops():
    """one DeviceOps per rank, each over a Context of its own (never Context.get).  A DeviceOps installs a side stream on a
    context that has none and runs torch and the C-ABI calls on it; a second DeviceOps on the same context would find the
    stream set and run torch work on another stream.  Own contexts also leave the shared context's stream alone.  Python
    cannot destroy a context, so the module makes MAX_RANKS of them once and trims their pools at the end."""
    from arrow_b200 import Context
    from arrow_b200 import distributed as d
    shared_stream = Context.get(0).stream
    ops = [d.DeviceOps(Context(0)) for _ in range(MAX_RANKS)]
    yield ops
    torch.cuda.synchronize()
    for o in ops:
        o.ctx.trim()
    assert Context.get(0).stream == shared_stream, "the shared context's stream changed"


@pytest.fixture(autouse=True)
def no_threads_left():
    before = threading.active_count()
    yield
    assert threading.active_count() == before, "a rank thread outlived its test"


def shard_bounds(n, world, rng, empty=()):
    """row ranges [lo, hi) in rank order: uneven lengths (weights in [1, 2), so no non-empty shard has fewer than
    n / (2 * world - 1) rows), and no rows on the ranks in `empty`"""
    w = np.where(np.isin(np.arange(world), list(empty)), 0.0, rng.uniform(1.0, 2.0, world))
    cuts = np.concatenate([[0], np.round(np.cumsum(w) / w.sum() * n)]).astype(np.int64)
    cuts[-1] = n
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world)]


def _upload(ops, arr):
    from arrow_b200 import DeviceArray
    return DeviceArray.from_arrow(arr, ops.ctx)


# ---------------------------------------------------------------------------------------------------------------------
# group_by_sum_count
# ---------------------------------------------------------------------------------------------------------------------
KEY_KINDS = ("int8_few", "int32_neg", "uint64_full", "float32", "float64_special")
VALUE_KINDS = ("int64", "uint64", "int32", "float64")
KEY_NULLS = ("none", "one_rank", "every_rank", "rank_all_null")
GROUPBY_ROWS = 100_003


def _key_column(kind, n, rng):
    if kind == "int8_few":              # two groups (and the null key): fewer groups than ranks for P >= 3
        return pa.int8(), np.array([-128, 127], np.int8)[rng.integers(0, 2, n)]
    if kind == "int32_neg":
        v = rng.integers(-3000, 3000, n).astype(np.int32)
        v[rng.random(n) < 0.01] = np.iinfo(np.int32).min
        v[rng.random(n) < 0.01] = np.iinfo(np.int32).max
        return pa.int32(), v
    if kind == "uint64_full":
        pool = np.concatenate([np.array([0, 1, 1 << 63, (1 << 64) - 1], np.uint64),
                               rng.integers(0, np.iinfo(np.uint64).max, 4000, np.uint64, endpoint=True)])
        return pa.uint64(), pool[rng.integers(0, len(pool), n)]
    if kind == "float32":
        pool = np.concatenate([(rng.standard_normal(3000) * 1000).astype(np.float32), er.special_values(np.float32)])
        return pa.float32(), pool[rng.integers(0, len(pool), n)]
    # float64: +-0, NaNs of several payloads, +-inf and the least subnormal are keys of their own, and frequent
    sp = er.special_values(np.float64)
    pool = rng.standard_normal(2000) * 1e6
    v = pool[rng.integers(0, len(pool), n)]
    pick = rng.random(n) < 0.3
    v[pick] = sp[rng.integers(0, len(sp), int(pick.sum()))]
    return pa.float64(), v


def _value_column(kind, gid, rng):
    """values of the kind; a float64 group's class (all finite, with a NaN, with +inf, with both infinities, all -0.0)
    follows its id, so the NaN / inf outcomes do not depend on how many rows a group has"""
    n = len(gid)
    if kind in ("int64", "uint64", "int32"):
        dt = np.dtype(kind)
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        v[rng.random(n) < 0.02] = info.max
        v[rng.random(n) < 0.02] = info.min
        return pa.from_numpy_dtype(dt), v
    v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)
    cls = gid % 7
    one = rng.random(n) < 0.05
    v[(cls == 1) & one] = np.array([np.nan, -np.nan, er.special_values(np.float64)[4]])[rng.integers(0, 3, n)][(cls == 1) & one]
    v[(cls == 2) & one] = np.inf
    v[(cls == 3) & one] = np.where(rng.random(n) < 0.5, np.inf, -np.inf)[(cls == 3) & one]
    v[cls == 4] = -0.0
    v[(cls == 5) & one] = er.special_values(np.float64)[-1]        # the least subnormal
    return pa.float64(), v


def _group_ids(kt, kv, kvalid):
    """group id of every row by the key's bits, the null key last"""
    kb = np.where(kvalid, kv.view(er.UINT_OF_WIDTH[kv.dtype.itemsize]).astype(np.uint64), 0)
    uniq, inv = np.unique(kb[kvalid], return_inverse=True)
    gid = np.full(len(kv), len(uniq), np.int64)
    gid[kvalid] = inv
    groups = [(True, int(b)) for b in uniq.tolist()] + ([(False, 0)] if (~kvalid).any() else [])
    return gid, groups


def groupby_case(key_kind, value_kind, key_nulls, world, seed):
    rng = np.random.default_rng(seed)
    n = GROUPBY_ROWS
    bounds = shard_bounds(n, world, rng, empty={1} if world >= 3 else ())
    kt, kv = _key_column(key_kind, n, rng)
    holders = [r for r, (lo, hi) in enumerate(bounds) if hi > lo]
    kvalid = np.ones(n, bool)
    if key_nulls == "every_rank":
        kvalid = rng.random(n) >= 0.05
    elif key_nulls in ("one_rank", "rank_all_null"):     # a rank other than 0: the null group has to travel to rank 0
        lo, hi = bounds[holders[-1]]
        kvalid[lo:hi] = rng.random(hi - lo) >= 0.1 if key_nulls == "one_rank" else False
    gid, groups = _group_ids(kt, kv, kvalid)
    vt, vv = _value_column(value_kind, gid, rng)
    vvalid = rng.random(n) >= 0.1
    vvalid[gid == 0] = False                              # a group whose every value is null: count 0, null sum
    lo, hi = bounds[holders[0]]
    vvalid[lo:hi][gid[lo:hi] == len(groups) - 1] = False  # one with no valid value on one rank: a partial with count 0
    keys, values = sort_ref.to_arrow(kt, kv, kvalid), sort_ref.to_arrow(vt, vv, vvalid)
    return keys, values, bounds, gid, groups


def groupby_reference(values, gid, n_groups):
    """per group: (count, exact sum) -- an int wrapped to the sum type, or a float (NaN / +-inf class decided from the
    specials, else math.fsum) with the sum of |x| for the error bound; the sum is None where the count is 0"""
    ok = er.valid_mask(values)
    v, g = er.raw(values)[ok], gid[ok]
    counts = np.bincount(g, minlength=n_groups)
    if pa.types.is_integer(values.type):
        signed = not pa.types.is_uint64(values.type)
        sums = [er.wrap64(x, signed) for x in er.exact_int_sums(g, v, n_groups)]
        return counts, sums, None
    nan = np.bincount(g, weights=np.isnan(v), minlength=n_groups) > 0
    pinf = np.bincount(g, weights=v == np.inf, minlength=n_groups) > 0
    ninf = np.bincount(g, weights=v == -np.inf, minlength=n_groups) > 0
    fin = np.isfinite(v)
    fs = er.fsums(g[fin], v[fin], n_groups)
    absum = np.bincount(g[fin], weights=np.abs(v[fin]), minlength=n_groups)
    sums = [math.nan if a or (b and c) else (math.inf if b else (-math.inf if c else s))
            for a, b, c, s in zip(nan.tolist(), pinf.tolist(), ninf.tolist(), fs)]
    return counts, sums, absum


def check_groupby(outs, keys, values, gid, groups, world):
    counts, sums, absum = groupby_reference(values, gid, len(groups))
    index = {g: i for i, g in enumerate(groups)}
    seen = np.zeros(len(groups), bool)
    for rank, (k, s, c) in enumerate(outs):
        assert k.type == keys.type and len(k) == len(s) == len(c)
        kvalid, kb = er.valid_mask(k), er.bits(k).astype(np.uint64)
        owner = (fmix64_np(kb) % np.uint64(world)).astype(np.int64)
        wrong = np.flatnonzero(np.where(kvalid, owner, 0) != rank)
        assert len(wrong) == 0, f"rank {rank} holds keys it does not own: {[k[int(i)] for i in wrong[:5]]}"
        for i, (ok, b, sum_, cnt) in enumerate(zip(kvalid.tolist(), kb.tolist(), s.to_pylist(), c.to_pylist())):
            g = index.get((ok, b if ok else 0))
            assert g is not None, f"rank {rank}: key {k[i]} (bits {b:#x}) is not in the input"
            assert not seen[g], f"key {k[i]} (bits {b:#x}) appears twice"
            seen[g] = True
            want_c, want_s = int(counts[g]), sums[g]
            assert cnt == want_c, f"key {k[i]}: count {cnt} != {want_c}"
            if want_c == 0:
                assert sum_ is None, f"key {k[i]}: sum {sum_} where every value is null"
            elif absum is None:
                assert sum_ == want_s, f"key {k[i]}: sum {sum_} != {want_s}"
            elif math.isnan(want_s) or math.isinf(want_s):
                assert er.same_value(sum_, want_s), f"key {k[i]}: sum {sum_} != {want_s}"
            else:
                tol = (want_c - 1) * 2.0 ** -53 * absum[g]
                assert math.isfinite(sum_) and abs(sum_ - want_s) <= tol, f"key {k[i]}: sum {sum_} != {want_s} (tolerance {tol})"
    missing = np.flatnonzero(~seen)
    assert len(missing) == 0, f"{len(missing)} groups missing, e.g. {[groups[int(i)] for i in missing[:5]]}"


@pytest.mark.parametrize("key_nulls", KEY_NULLS)
@pytest.mark.parametrize("key_kind", KEY_KINDS)
@pytest.mark.parametrize("world", WORLDS)
def test_group_by_sum_count_matches_exact_sums(rank_ops, world, key_kind, key_nulls):
    from arrow_b200 import distributed as d
    for vi, value_kind in enumerate(VALUE_KINDS):
        keys, values, bounds, gid, groups = groupby_case(key_kind, value_kind, key_nulls, world,
                                                         SEED + 1000 * world + 100 * KEY_KINDS.index(key_kind) + 10 * vi)

        def rank_fn(rank, xchg):
            ops = rank_ops[rank]
            lo, hi = bounds[rank]
            out = d.group_by_sum_count(_upload(ops, keys.slice(lo, hi - lo)), _upload(ops, values.slice(lo, hi - lo)), ops, xchg)
            return tuple(x.to_arrow() for x in out)

        outs = run_ranks(world, rank_fn)
        check_groupby(outs, keys, values, gid, groups, world)


# ---------------------------------------------------------------------------------------------------------------------
# sort_indices
# ---------------------------------------------------------------------------------------------------------------------
SORT_PATTERNS = ("none", "p10", "rank_all_null", "all_null", "sparse_off_grid", "all_equal", "empty_shards")
SAMPLES = (1, 3, 4096)


def _sort_rows(world):
    """enough rows that every shard is longer than 4096 (shard_bounds keeps each above n / (2 * world - 1)), so that even
    4096 samples per rank leave rows off an evenly spaced grid"""
    return 4500 * (2 * world - 1) + world


def sort_case(t, pattern, world, samples, seed):
    rng = np.random.default_rng(seed)
    n = _sort_rows(world)
    bounds = shard_bounds(n, world, rng, empty=set(range(0, world, 2)) if pattern == "empty_shards" else ())
    v = sort_ref.edge_values(t, n, rng)
    if pattern == "all_equal":
        v[:] = v[0]
    valid = rng.random(n) >= 0.1
    if pattern == "none":
        valid[:] = True
    elif pattern == "all_null":
        valid[:] = False
    elif pattern == "rank_all_null":
        lo, hi = bounds[world // 2]
        valid[lo:hi] = False
    elif pattern == "sparse_off_grid":
        # no valid row where a sampler that takes every step-th row of the shard and then drops the nulls would look
        # (step = ceil(shard rows / samples)): only a sampler that looks among the valid rows finds any splitter
        for lo, hi in bounds:
            step = -(-(hi - lo) // samples)
            assert step >= 2
            valid[lo:hi] &= np.arange(hi - lo) % step != 0
            valid[lo:hi] &= rng.random(hi - lo) < 0.3
    return sort_ref.to_arrow(t, v, valid), bounds


def check_sort(outs, arr, bounds, return_keys):
    n = len(arr)
    valid = er.valid_mask(arr)
    ref = sort_ref.sort_indices_np(arr)
    n_valid = int(valid.sum())
    segs = [o[0] for o in outs]
    nulls = [o[1] for o in outs]
    for rank, (lo, hi) in enumerate(bounds):
        assert segs[rank].dtype == np.int64 and nulls[rank].dtype == np.int64
        assert np.array_equal(nulls[rank], lo + np.flatnonzero(~valid[lo:hi])), f"rank {rank}: null segment is not its own null rows"
    # ties get one rank: NaNs tie, -0.0 ties +0.0
    sv = er.raw(arr)[ref[:n_valid]]
    same = sv[1:] == sv[:-1]
    if np.issubdtype(sv.dtype, np.floating):
        same |= np.isnan(sv[1:]) & np.isnan(sv[:-1])
    key_rank = np.zeros(n, np.int64)
    key_rank[ref[:n_valid]] = np.concatenate([[0], np.cumsum(~same)])
    held = [r for r in range(len(segs)) if len(segs[r])]
    for a, b in zip(held, held[1:]):
        assert key_rank[segs[a]].max() <= key_rank[segs[b]].min(), f"rank {a} holds a key that sorts after one on rank {b}"
    got = np.concatenate(segs + nulls)
    assert len(got) == n, f"{len(got)} rows out of {n}"
    bad = np.flatnonzero(got != ref)
    assert len(bad) == 0, f"{len(bad)} positions differ from the single-process sort, first at {bad[:5].tolist()}: " \
                          f"got rows {got[bad[:5]].tolist()} want {ref[bad[:5]].tolist()}; value segment sizes {[len(s) for s in segs]}"
    if return_keys:
        bits = er.bits(arr)
        for rank, o in enumerate(outs):
            got_bits = o[2].view(er.UINT_OF_WIDTH[o[2].dtype.itemsize])
            assert np.array_equal(got_bits, bits[segs[rank]]), f"rank {rank}: returned keys are not the sorted values' bits"


@pytest.mark.parametrize("return_keys", [False, True], ids=["payload", "keys"])
@pytest.mark.parametrize("samples", SAMPLES)
@pytest.mark.parametrize("pattern", SORT_PATTERNS)
@pytest.mark.parametrize("world", WORLDS)
def test_sort_indices_matches_single_process_sort(rank_ops, world, pattern, samples, return_keys):
    from arrow_b200 import distributed as d
    for ti, t in enumerate(sort_ref.NUMERIC):
        arr, bounds = sort_case(t, pattern, world, samples,
                                SEED + 100_000 * world + 1000 * SORT_PATTERNS.index(pattern) + 10 * ti + samples)

        def rank_fn(rank, xchg):
            ops = rank_ops[rank]
            lo, hi = bounds[rank]
            out = d.sort_indices(_upload(ops, arr.slice(lo, hi - lo)), ops, xchg, samples_per_rank=samples, return_keys=return_keys)
            return tuple(x.cpu().numpy() for x in out)

        outs = run_ranks(world, rank_fn)
        check_sort(outs, arr, bounds, return_keys)
