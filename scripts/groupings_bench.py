#!/usr/bin/env python
"""Group-major order and the list-valued hash aggregates at config 3's size.  Legs:
  make_groupings over `--rows` ids from the Grouper over uniform int64 keys in `--groups` groups (3 radix passes),
  make_groupings over `--rows` ids in 200 groups (1 pass),
  hash_list over float64 with 10% nulls, `--groups` groups (resize + consume + finalize),
  hash_distinct over int32 values in [0, 64), `--distinct-groups` groups (resize + consume + finalize).
Legs alternate round by round in one process; CUDA-event times, median of `--reps` rounds after one warm-up round.  One
JSON line per leg with the card, its power limit, ms, the algorithmic bytes (inputs read once, outputs written once) and
their share of 3.35 TB/s, and parity_ok: the leg's output against a torch restatement from the same run
(torch.sort(ids, stable=True) for the rows; the per-group sets of (group, value) pairs for hash_distinct)."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyarrow as pa
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000_000)
ap.add_argument("--groups", type=int, default=10_000_000)
ap.add_argument("--distinct-groups", type=int, default=1_000_000)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
n = args.rows
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(0x0FF1CE)


def view(arr: DeviceArray, dtype, length=None, buffer=1):
    """zero-copy torch view of one of a DeviceArray's buffers"""
    length = len(arr) if length is None else length

    class _Cai:
        pass
    shim = _Cai()
    shim.__cuda_array_interface__ = {"shape": (length,), "typestr": {torch.int32: "<i4", torch.float64: "<f8",
                                                                     torch.uint8: "|u1"}[dtype],
                                     "data": (arr.buffers[buffer].ptr, False), "version": 2}
    return torch.as_tensor(shim, device="cuda")


def grouper_ids(groups):
    keys_t = torch.randint(0, groups, (n,), dtype=torch.int64, device="cuda", generator=gen)
    torch.cuda.synchronize()
    g = bc.Grouper([pa.int64()], ctx)
    ids = g.consume(DeviceArray.from_pointers(ctx, pa.int64(), n, keys_t.data_ptr()))
    ctx.sync()
    return ids, g.num_groups


ids_many, g_many = grouper_ids(args.groups)
ids_few, g_few = grouper_ids(200)
ids_dist, g_dist = grouper_ids(args.distinct_groups)
f64_t = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
valid_t = torch.rand(n, device="cuda", generator=gen) >= 0.1
bits_t = torch.zeros((n + 7) // 8 + 8, dtype=torch.uint8, device="cuda")
weights = (1 << torch.arange(8, device="cuda", dtype=torch.int32)).to(torch.uint8)
for lo in range(0, n, 1 << 27):
    m = min(1 << 27, n - lo)
    m8 = (m + 7) // 8 * 8
    v = torch.zeros(m8, dtype=torch.bool, device="cuda")
    v[:m] = valid_t[lo:lo + m]
    bits_t[lo // 8: lo // 8 + m8 // 8] = (v.view(-1, 8).to(torch.uint8) * weights).sum(dim=1, dtype=torch.uint8)
del v
i32_t = torch.randint(0, 64, (n,), dtype=torch.int32, device="cuda", generator=gen)
torch.cuda.synchronize()
f64 = DeviceArray.from_pointers(ctx, pa.float64(), n, f64_t.data_ptr(), validity_ptr=bits_t.data_ptr(),
                                null_count=int((~valid_t).sum().item()))
i32 = DeviceArray.from_pointers(ctx, pa.int32(), n, i32_t.data_ptr())


def aggregate(fn, values, ids, groups):
    def go():
        agg = bc.HashAggregator(fn, values.type, ctx=ctx)
        agg.resize(groups)
        agg.consume(values, ids)
        return agg.finalize()
    return go


def rows_parity(out, ids, groups):
    ids_t = view(ids, torch.int32)
    want = torch.sort(ids_t, stable=True).indices
    ok = torch.equal(view(out.children[0], torch.int32).to(torch.int64), want)
    del want
    offs = torch.zeros(groups + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(torch.bincount(ids_t, minlength=groups), 0)
    return ok and torch.equal(view(out, torch.int32, groups + 1).to(torch.int64), offs)


def list_parity(out, ids, groups):
    perm = torch.sort(view(ids, torch.int32), stable=True).indices
    child = out.children[0]
    got_valid = torch.ones(n, dtype=torch.bool, device="cuda") if child.buffers[0] is None else \
        ((view(child, torch.uint8, (n + 7) // 8, 0)[:, None] >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1
         ).to(torch.bool).view(-1)[:n]
    want_valid = valid_t[perm]
    ok = torch.equal(got_valid, want_valid)
    ok = ok and torch.equal(view(child, torch.float64)[want_valid], f64_t[perm][want_valid])
    return ok and rows_parity_offsets(out, ids, groups)


def rows_parity_offsets(out, ids, groups):
    offs = torch.zeros(groups + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(torch.bincount(view(ids, torch.int32), minlength=groups), 0)
    return torch.equal(view(out, torch.int32, groups + 1).to(torch.int64), offs)


def distinct_parity(out, ids, groups):
    want = torch.unique(view(ids, torch.int32).to(torch.int64) * 64 + i32_t)
    offs = view(out, torch.int32, groups + 1).to(torch.int64)
    sizes = offs[1:] - offs[:-1]
    group_of = torch.repeat_interleave(torch.arange(groups, device="cuda"), sizes)
    got = torch.sort(group_of * 64 + view(out.children[0], torch.int32, int(offs[-1].item()))).values
    return torch.equal(got, want)


# (name, callable, groups, algorithmic bytes, parity check)
legs = [
    (f"make_groupings {g_many} groups", lambda: bc.Grouper.make_groupings(ids_many, g_many), g_many, 8 * n + 4 * g_many,
     lambda o: rows_parity(o, ids_many, g_many)),
    (f"make_groupings {g_few} groups", lambda: bc.Grouper.make_groupings(ids_few, g_few), g_few, 8 * n + 4 * g_few,
     lambda o: rows_parity(o, ids_few, g_few)),
    ("hash_list float64 null_p 0.1", aggregate("hash_list", f64, ids_many, g_many), g_many,
     int(n * (8 + 4 + 0.25)) + 4 * g_many, lambda o: list_parity(o, ids_many, g_many)),
    ("hash_distinct int32 in [0, 64)", aggregate("hash_distinct", i32, ids_dist, g_dist), g_dist, None,
     lambda o: distinct_parity(o, ids_dist, g_dist)),
]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    del out
    return e0.elapsed_time(e1)


times = {leg[0]: [] for leg in legs}
for rnd in range(args.reps + 1):
    for name, fn, *_ in legs:
        t = timed(fn)
        if rnd:
            times[name].append(t)
parity = {}
for name, fn, _, _, check in legs:
    out = fn()
    ctx.sync()
    ctx.trim()  # hand the pool's cached blocks back: the torch restatement needs the memory
    parity[name] = bool(check(out))
    del out
    torch.cuda.empty_cache()

gpu = torch.cuda.get_device_name(0)
try:
    import pynvml
    pynvml.nvmlInit()
    power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000
except Exception:
    power = None
for name, _, groups, nbytes, _ in legs:
    ms = statistics.median(times[name])
    print(json.dumps({"leg": name, "rows": n, "groups": groups, "median_ms": round(ms, 3),
                      "min_ms": round(min(times[name]), 3), "max_ms": round(max(times[name]), 3), "alg_bytes": nbytes,
                      "share_of_3.35TBps": None if nbytes is None else round(nbytes / (ms * 1e-3) / 3.35e12, 3),
                      "gpu": gpu, "power_limit_w": power, "parity_ok": parity[name]}), flush=True)
