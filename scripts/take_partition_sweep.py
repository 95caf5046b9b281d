#!/usr/bin/env python
"""Direct vs partitioned random Take (selection_take.cu take_partition_plan, take_partitioned.cu), alternated in one
process through B2_TAKE_PARTITION=0|1 (read on every call).

  --ab N     : b2_take_cast_arith at the bench shape (float64 values, int64 uniform random indices, null_p 0.1, `--rows`
               rows), N rounds per arm after a warm-up, alternating; median and spread of each arm, null counts compared.
  --sweep    : crossover grid, table size (64 MB .. 8 GB of float64) x rows, best of 3 per arm, for the plan thresholds.
CUDA-event times.  One JSON line per measurement."""
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
from bench import SEED, make_validity

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000_000)
ap.add_argument("--ab", type=int, default=0)
ap.add_argument("--sweep", action="store_true")
args = ap.parse_args()
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    nulls = out.null_count
    del out
    return e0.elapsed_time(e1), nulls


def inputs(n_values, n, gen):
    values_t = torch.rand(n_values, dtype=torch.float64, device="cuda", generator=gen) * 1e6
    vvalid_t, v_nulls = make_validity(torch, n_values, gen)
    idx_t = torch.randint(0, n_values, (n,), dtype=torch.int64, device="cuda", generator=gen)
    other_t = torch.rand(n, dtype=torch.float32, device="cuda", generator=gen) * 1e6
    ovalid_t, o_nulls = make_validity(torch, n, gen)
    torch.cuda.synchronize()
    keep = (values_t, vvalid_t, idx_t, other_t, ovalid_t)
    values = DeviceArray.from_pointers(ctx, pa.float64(), n_values, values_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)
    idx = DeviceArray.from_pointers(ctx, pa.int64(), n, idx_t.data_ptr())
    other = DeviceArray.from_pointers(ctx, pa.float32(), n, other_t.data_ptr(), validity_ptr=ovalid_t.data_ptr(), null_count=o_nulls)
    return keep, values, idx, other


def arm(partition, fn):
    os.environ["B2_TAKE_PARTITION"] = partition
    return timed(fn)


gen = torch.Generator(device="cuda")
gen.manual_seed(SEED)
if args.ab:
    n = args.rows
    keep, values, idx, other = inputs(n, n, gen)
    fused = lambda: bc.take_cast_arith(values, idx, pa.float32(), "add", other)  # noqa: E731
    for p in ("0", "1"):
        arm(p, fused)
    times, nulls = {"0": [], "1": []}, {"0": set(), "1": set()}
    for _ in range(args.ab):
        for p in ("0", "1"):
            t, nn = arm(p, fused)
            times[p].append(t)
            nulls[p].add(nn)
    for p in ("0", "1"):
        ts = sorted(times[p])
        print(json.dumps({"call": "b2_take_cast_arith", "rows": n, "partition": p, "median_ms": round(statistics.median(ts), 3),
                          "min_ms": round(ts[0], 3), "max_ms": round(ts[-1], 3), "rounds": len(ts),
                          "null_counts": sorted(nulls[p])}), flush=True)
    take = lambda: bc.take(values, idx)  # noqa: E731
    for p in ("0", "1"):
        arm(p, take)
        best = min(arm(p, take)[0] for _ in range(3))
        print(json.dumps({"call": "b2_take", "rows": n, "partition": p, "best_ms": round(best, 3)}), flush=True)
    del keep, values, idx, other
    torch.cuda.empty_cache()

if args.sweep:
    for table_mb in (64, 256, 1024, 4096, 8192):
        for n in (1 << 22, 1 << 24, 1 << 26, 1 << 28, 1_000_000_000):
            keep, values, idx, other = inputs(table_mb << 17, n, gen)
            fused = lambda: bc.take_cast_arith(values, idx, pa.float32(), "add", other)  # noqa: E731
            row = {"table_mb": table_mb, "rows": n}
            for p in ("0", "1"):
                arm(p, fused)
                row["ms_partition_" + p] = round(min(arm(p, fused)[0] for _ in range(3)), 3)
            print(json.dumps(row), flush=True)
            del keep, values, idx, other
            torch.cuda.empty_cache()
