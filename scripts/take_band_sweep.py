#!/usr/bin/env python
"""Sweep of B2_TAKE_BAND_MB (selection_take.cu take_bands): take / fused take+cast+add at the benchmarked size with the
values' validity bitmap probed in bands of the given size (0 = one band, the round-1 kernel).  CUDA-event times, best of
3 after a warm-up; null counts must agree across band sizes.  One JSON line per band size."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyarrow as pa
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray
from bench import SEED, make_validity

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000_000)
ap.add_argument("--bands", default="0,24,32,40,48,64")
args = ap.parse_args()
n = args.rows
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(SEED)
values_t = torch.rand(n, dtype=torch.float64, device="cuda", generator=gen) * 1e6
vvalid_t, v_nulls = make_validity(torch, n, gen)
idx_t = torch.randint(0, n, (n,), dtype=torch.int64, device="cuda", generator=gen)
idx32_t = idx_t.to(torch.int32)
other_t = torch.rand(n, dtype=torch.float32, device="cuda", generator=gen) * 1e6
ovalid_t, o_nulls = make_validity(torch, n, gen)
torch.cuda.synchronize()
values = DeviceArray.from_pointers(ctx, pa.float64(), n, values_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)
idx = DeviceArray.from_pointers(ctx, pa.int64(), n, idx_t.data_ptr())
idx32 = DeviceArray.from_pointers(ctx, pa.int32(), n, idx32_t.data_ptr())
other = DeviceArray.from_pointers(ctx, pa.float32(), n, other_t.data_ptr(), validity_ptr=ovalid_t.data_ptr(), null_count=o_nulls)


def timed(fn, reps=3):
    best, nulls = None, None
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        nulls = out.null_count
        del out
        if r:
            t = e0.elapsed_time(e1)
            best = t if best is None else min(best, t)
    return round(best, 3), nulls


def pipeline_tail(reps=3):
    """cast + add right after a take: what the take leaves behind in L2 (evict_last lines) is their problem"""
    best = None
    for r in range(reps + 1):
        t = bc.take(values, idx)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        c = bc.cast(t, pa.float32(), safe=False)
        o = bc.add(c, other)
        e1.record()
        e1.synchronize()
        del t, c, o
        if r:
            ms = e0.elapsed_time(e1)
            best = ms if best is None else min(best, ms)
    return round(best, 3)


inc = torch.randint(0, 3, (n,), dtype=torch.int64, device="cuda", generator=gen)
mono_t = torch.clamp(torch.cumsum(inc, 0), max=n - 1)
del inc
mono = DeviceArray.from_pointers(ctx, pa.int64(), n, mono_t.data_ptr())

for b in args.bands.split(","):
    os.environ["B2_TAKE_BAND_MB"] = b
    t_mono, _ = timed(lambda: bc.take(values, mono))
    t_tail = pipeline_tail()
    print(json.dumps({"band_mb": b, "take_monotonic_ms": t_mono, "cast_add_after_take_ms": t_tail}), flush=True)
    t_take, n_take = timed(lambda: bc.take(values, idx))
    t_take32, n_take32 = timed(lambda: bc.take(values, idx32))
    t_fused, n_fused = timed(lambda: bc.take_cast_arith(values, idx, pa.float32(), "add", other))
    print(json.dumps({"band_mb": b, "rows": n, "take_ms": t_take, "take_idx32_ms": t_take32, "fused_ms": t_fused,
                      "take_nulls": n_take, "take_idx32_nulls": n_take32, "fused_nulls": n_fused}), flush=True)
