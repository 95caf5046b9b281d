"""The packed states of the fused group-by and of hash_sum over group ids at their field limits, against an exact
reference (tests/packed_regimes.py): value fields filled to their last bit, the max-count guard's drain, values on and one
step past a sampled window's edges at rows the sample skips, compact tuples of exactly 64 bits on both sides of the
NARROW edge, dense key bands, and keys at their type's ends.  Every fused case also asserts path_counts() against the
restated path, and every hash_sum case the kernels it launched against the restated kernel list, so a case that drifts off
the regime it is named for fails instead of passing on another path."""
import numpy as np
import pyarrow as pa
import pytest

import arrow_b200.compute as bc
from arrow_b200 import DeviceArray, _cabi

from . import packed_regimes as P

pytestmark = pytest.mark.gpu

FUSED = P.fused_cases()
BYID = P.byid_cases()


def _device(ctx, values, valid, t):
    return DeviceArray.from_arrow(pa.array(values, t, mask=None if valid is None else ~valid), ctx)


@pytest.mark.parametrize("case", FUSED, ids=[c.name for c in FUSED])
def test_fused_group_by_packed_edges(ctx, case, monkeypatch):
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    batches = case.make()
    plans, _ = case.plans(batches)
    assert [p.path for p in plans] == case.paths, [p.why for p in plans]
    g = bc.GroupBySumCount(case.key_type, case.value_type, expected_groups=case.hint, ctx=ctx)
    want_paths = {"dense": 0, "compact": 0, "general": 0, "atomic": 0}
    for b, p in zip(batches, plans):
        g.consume(_device(ctx, b.keys, b.kvalid, case.key_type), _device(ctx, b.vals, b.vvalid, case.value_type))
        want_paths[p.path] += 1
        assert g.path_counts() == want_paths
    k, s, c = [x.to_arrow() for x in g.finalize()]
    got = pa.table({"k": k, "sum": s, "count": c}).sort_by("k")
    cat = lambda xs: None if all(x is None for x in xs) else np.concatenate(
        [np.ones(len(b.keys), bool) if x is None else x for x, b in zip(xs, batches)])
    want = P.group_sum_count(np.concatenate([b.keys for b in batches]), cat([b.kvalid for b in batches]),
                             np.concatenate([b.vals for b in batches]), cat([b.vvalid for b in batches]),
                             case.key_type, case.value_type)
    for col in ("k", "count", "sum"):
        gc, wc = got[col].combine_chunks(), want[col].combine_chunks()
        if not gc.equals(wc):
            bad = np.nonzero(~np.asarray(pa.compute.equal(gc, wc).fill_null(False)))[0][:5]
            raise AssertionError(f"{col}: {len(gc)} vs {len(wc)} rows; first differences at {bad}: "
                                 f"{gc.take(bad).to_pylist()} != {wc.take(bad).to_pylist()}")


@pytest.mark.parametrize("case", BYID, ids=[c.name for c in BYID])
def test_hash_sum_by_id_packed_edges(ctx, case, monkeypatch):
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    consumes = case.make()
    plans, _ = case.plans(consumes)
    assert [p.dense is not None for p in plans] == case.dense, [p.why for p in plans]
    agg = bc.HashAggregator("hash_sum", case.value_type, ctx=ctx)
    agg.resize(case.num_groups)
    lib = _cabi.lib()
    vw = case.value_type.bit_width // 8
    arrays = {}
    for (ids, vals, vvalid, off), p in zip(consumes, plans):
        key = (id(ids), id(vals))
        if key not in arrays:  # one device copy per array pair: later consumes slice it at other offsets
            arrays[key] = (_device(ctx, ids, None, pa.uint32()), _device(ctx, vals, vvalid, case.value_type))
        dids, dv = arrays[key]
        before = lib.b2_launch_count()
        agg.consume(dv.slice(off), dids.slice(off))
        assert lib.b2_launch_count() - before == p.launches(vw, len(ids) - off, case.num_groups), p.why
    got = agg.finalize().to_arrow()
    all_ids = np.concatenate([i[o:] for i, _, _, o in consumes])
    all_vals = np.concatenate([v[o:] for _, v, _, o in consumes])
    all_valid = None if all(vv is None for *_, vv, _ in consumes) else np.concatenate(
        [np.ones(len(i) - o, bool) if vv is None else vv[o:] for i, _, vv, o in consumes])
    want = P.sum_by_id(all_ids, all_vals, all_valid, case.num_groups, case.value_type)
    assert got.equals(want)
