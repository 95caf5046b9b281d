#!/usr/bin/env python
"""Variance-family aggregates at config 3's shape: `--rows` rows in `--groups` groups (uniform random int64 keys, ids
from the Grouper, not timed).  Times consume + finalize of
  hash_variance over int32 (exact path), float64 and int64 (two-pass), hash_kurtosis over float64,
  hash_sum + hash_count over the same float64 values (for comparison),
and the ungrouped variance over float64 and int32 next to bc.sum (b2_reduce).  A grouped leg's time includes creating the
aggregator and zeroing its state, as a caller pays it.  Legs alternate round by round in one
process; CUDA-event times, median of `--reps` rounds after one warm-up round.  One JSON line per leg with the card, its
power limit, ms, the algorithmic bytes (the reads the algorithm cannot avoid: ids + values once per pass, state written
once) and their share of 3.35 TB/s."""
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
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
n, G = args.rows, args.groups
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(0x0FF1CE)

keys_t = torch.randint(0, G, (n,), dtype=torch.int64, device="cuda", generator=gen)
torch.cuda.synchronize()
grouper = bc.Grouper([pa.int64()], ctx)
ids = grouper.consume(DeviceArray.from_pointers(ctx, pa.int64(), n, keys_t.data_ptr()))
groups = grouper.num_groups
del keys_t
f64_t = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen).mul_(100).add_(1e4)
i32_t = torch.randint(-2**31, 2**31 - 1, (n,), dtype=torch.int32, device="cuda", generator=gen)
i64_t = torch.randint(-2**40, 2**40, (n,), dtype=torch.int64, device="cuda", generator=gen)
torch.cuda.synchronize()
cols = {"float64": DeviceArray.from_pointers(ctx, pa.float64(), n, f64_t.data_ptr()),
        "int32": DeviceArray.from_pointers(ctx, pa.int32(), n, i32_t.data_ptr()),
        "int64": DeviceArray.from_pointers(ctx, pa.int64(), n, i64_t.data_ptr())}
width = {"float64": 8, "int32": 4, "int64": 8}


def grouped(fns, col):
    def go():
        out = []
        for fn in fns:
            agg = bc.HashAggregator(fn, cols[col].type, ctx=ctx)
            agg.resize(groups)
            agg.consume(cols[col], ids)
            out.append(agg.finalize())
        return out
    return go


def ungrouped(fn, col):
    return lambda: getattr(bc, fn)(cols[col])


# (name, callable, passes over ids + values, state bytes per group written once)
legs = [
    ("hash_variance int32 (exact)", grouped(["hash_variance"], "int32"), 1, "int32", True, 40),
    ("hash_variance float64 (two-pass)", grouped(["hash_variance"], "float64"), 2, "float64", True, 40),
    ("hash_variance int64 (two-pass)", grouped(["hash_variance"], "int64"), 2, "int64", True, 40),
    ("hash_kurtosis float64 (two-pass)", grouped(["hash_kurtosis"], "float64"), 2, "float64", True, 40),
    ("hash_sum + hash_count float64", grouped(["hash_sum", "hash_count"], "float64"), 2, "float64", True, 16),
    ("variance float64", ungrouped("variance", "float64"), 2, "float64", False, 0),
    ("variance int32 (exact)", ungrouped("variance", "int32"), 1, "int32", False, 0),
    ("sum float64 (b2_reduce)", ungrouped("sum", "float64"), 1, "float64", False, 0),
    ("sum int32 (b2_reduce)", ungrouped("sum", "int32"), 1, "int32", False, 0),
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

gpu = torch.cuda.get_device_name(0)
try:
    import pynvml
    pynvml.nvmlInit()
    power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000
except Exception:
    power = None
for name, _, passes, col, with_ids, state in legs:
    per_row = width[col] + (4 if with_ids else 0)
    nbytes = passes * n * per_row + groups * state
    ms = statistics.median(times[name])
    print(json.dumps({"leg": name, "rows": n, "groups": groups if with_ids else 1, "median_ms": round(ms, 3),
                      "min_ms": round(min(times[name]), 3), "max_ms": round(max(times[name]), 3), "alg_bytes": nbytes,
                      "share_of_3.35TBps": round(nbytes / (ms * 1e-3) / 3.35e12, 3), "gpu": gpu, "power_limit_w": power}),
          flush=True)
