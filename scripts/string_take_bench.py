#!/usr/bin/env python
"""Random Take on a large_utf8 column: `--rows` strings of 0-32 B (null_p 0.1, the shape of bench.py's c5 filter input),
gathered by as many uniform random int64 indices.  CUDA-event times of whole b2_take calls after one warm-up call; one
JSON line with the median / min / max, the card and its power limit.  With --digest the line also carries a SHA-256 of the
result's offsets, bytes and validity, so two builds can be checked to produce byte-identical output on the same seed."""
import argparse
import hashlib
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyarrow as pa
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray
from bench import SEED, _view, make_validity

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=500_000_000)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--digest", action="store_true")
args = ap.parse_args()
m = args.rows
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(SEED)

lens = torch.randint(0, 33, (m,), dtype=torch.int64, device="cuda", generator=gen)
offs = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
torch.cumsum(lens, 0, out=offs[1:])
total = int(offs[-1].item())
del lens
data = torch.randint(97, 123, (total + 64,), dtype=torch.uint8, device="cuda", generator=gen)
svalid_t, s_nulls = make_validity(torch, m, gen)
idx_t = torch.randint(0, m, (m,), dtype=torch.int64, device="cuda", generator=gen)
torch.cuda.synchronize()
strs = DeviceArray.from_pointers(ctx, pa.large_string(), m, offs.data_ptr(), validity_ptr=svalid_t.data_ptr(), null_count=s_nulls,
                                 data2_ptr=data.data_ptr())
idx = DeviceArray.from_pointers(ctx, pa.int64(), m, idx_t.data_ptr())


def timed():
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = bc.take(strs, idx)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def digest(res):
    """SHA-256 over the offsets, the value bytes and the validity bitmap (bits past the last row masked), 256 MB at a time"""
    h = hashlib.sha256()
    ro = torch.as_tensor(_view(res.buffers[1].ptr, res.length + 1, "<i8", res), device="cuda")
    n_bytes = int(ro[-1].item())
    parts = [(res.buffers[1].ptr, (res.length + 1) * 8), (res.buffers[2].ptr, n_bytes)]
    if res.buffers[0] is not None:
        parts.append((res.buffers[0].ptr, res.length // 8))
    for ptr, size in parts:
        for lo in range(0, size, 1 << 28):
            h.update(torch.as_tensor(_view(ptr + lo, min(1 << 28, size - lo), "|u1", res), device="cuda").cpu().numpy().tobytes())
    if res.buffers[0] is not None and res.length % 8:
        last = torch.as_tensor(_view(res.buffers[0].ptr + res.length // 8, 1, "|u1", res), device="cuda").item()
        h.update(bytes([last & ((1 << (res.length % 8)) - 1)]))
    return h.hexdigest()


_, out = timed()  # warm-up: the pool allocates the output buffers here
del out
times = []
for _ in range(args.reps):
    t, out = timed()
    times.append(t)
    null_count = out.null_count
    del out
line = {"call": "b2_take large_utf8", "rows": m, "mean_len": total / m, "indices": "uniform random int64", "null_p": 0.1,
        "median_ms": round(statistics.median(times), 3), "min_ms": round(min(times), 3), "max_ms": round(max(times), 3),
        "reps": len(times), "null_count": null_count, "gpu": torch.cuda.get_device_name(0)}
try:
    import pynvml
    pynvml.nvmlInit()
    line["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000
except Exception:
    line["power_limit_w"] = None
if args.digest:
    _, out = timed()
    line["sha256"] = digest(out)
    del out
print(json.dumps(line), flush=True)
