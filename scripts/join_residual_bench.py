#!/usr/bin/env python
"""Hash join with a residual filter, phase by phase: `--probe-rows` probe rows (int64 keys, `--match` of them matching)
against `--build-keys` keys with two build rows each, residual `l.v < r.w` over float64 payloads with 10 % nulls (about half
of the candidate pairs pass).  For INNER, LEFT OUTER, LEFT SEMI and FULL OUTER each round times
  candidate : bc.hash_join_indices(probe, build, "inner")           (b2_hash_join_ex)
  filter    : take of both payloads at the candidates + bc.less      (the caller's gather + compare)
  residual  : bc.join_residual(...)                                  (b2_join_residual)
with CUDA events; the median of `--reps` rounds after one warm-up round.  One JSON line per leg with the card, its power
limit, the residual step's algorithmic bytes (reads: 8 B per candidate, the keep bits, 4 B per left row for each scan of the
per-row counts; writes: the result) and a parity flag from invariants checked with torch on the candidates:
INNER rows = passing pairs, SEMI + ANTI = probe rows, LEFT OUTER rows = passing pairs + probe rows with none,
FULL OUTER rows = LEFT OUTER rows + build rows with none."""
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
ap.add_argument("--probe-rows", type=int, default=200_000_000)
ap.add_argument("--build-keys", type=int, default=10_000_000)
ap.add_argument("--match", type=float, default=0.8)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("join_residual_bench.py measures on a GPU; none is visible")
n_left = args.probe_rows // 8 * 8
n_keys = args.build_keys
n_right = 2 * n_keys
torch.cuda.set_device(0)
ctx = Context.get(0)
ctx.stream = torch.cuda.current_stream().cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(0x0FF1CE)


def packed(valid: torch.Tensor) -> torch.Tensor:
    """LSB-first validity bitmap of a bool tensor whose length is a multiple of 8"""
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device="cuda")
    return (valid.view(-1, 8).to(torch.uint8) * w).sum(1, dtype=torch.uint8)


def column(t: torch.Tensor, valid=None, bits=None) -> DeviceArray:
    typ = pa.int64() if t.dtype == torch.int64 else pa.float64()
    if valid is None:
        return DeviceArray.from_pointers(ctx, typ, t.numel(), t.data_ptr())
    return DeviceArray.from_pointers(ctx, typ, t.numel(), t.data_ptr(), validity_ptr=bits.data_ptr(),
                                     null_count=int((~valid).sum()))


class _View:  # a uint32 DeviceArray as a torch tensor (row numbers stay below 2^31 here)
    def __init__(self, a: DeviceArray):
        self.__cuda_array_interface__ = {"shape": (a.length,), "typestr": "<i4", "version": 3,
                                         "data": (a.buffers[1].ptr + 4 * a.offset if a.length else 0, False)}


def rows(a: DeviceArray) -> torch.Tensor:
    return torch.as_tensor(_View(a), device="cuda").to(torch.int64) if a.length else torch.zeros(0, dtype=torch.int64, device="cuda")


# build: every key twice, shuffled; probe: `match` of the rows draw a build key, the rest a key no build row has
build_keys = (torch.arange(n_keys, device="cuda", dtype=torch.int64) * 7 + 3).repeat(2)
build_keys = build_keys[torch.randperm(n_right, device="cuda", generator=gen)]
hit = torch.rand(n_left, device="cuda", generator=gen) < args.match
pick = torch.randint(0, n_keys, (n_left,), device="cuda", generator=gen, dtype=torch.int64)
probe_keys = torch.where(hit, pick * 7 + 3, pick * 7 + 5)
del hit, pick
lv = torch.randn(n_left, device="cuda", generator=gen, dtype=torch.float64)
rw = torch.randn(n_right, device="cuda", generator=gen, dtype=torch.float64)
lv_valid = torch.rand(n_left, device="cuda", generator=gen) >= 0.1
rw_valid = torch.rand(n_right, device="cuda", generator=gen) >= 0.1
lv_bits, rw_bits = packed(lv_valid), packed(rw_valid)
torch.cuda.synchronize()
d_lk, d_rk = column(probe_keys), column(build_keys)
d_lv, d_rw = column(lv, lv_valid, lv_bits), column(rw, rw_valid, rw_bits)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return out, e0.elapsed_time(e1)


LEGS = ["inner", "left outer", "left semi", "full outer"]
times = {leg: {"candidate": [], "filter": [], "residual": []} for leg in LEGS}
results = {}
for rnd in range(args.reps + 1):
    for leg in LEGS:
        (cl, cr), t_cand = timed(lambda: bc.hash_join_indices([d_lk], [d_rk], "inner"))
        keep, t_filt = timed(lambda: bc.less(bc.take(d_lv, cl), bc.take(d_rw, cr)))
        (ol, orr), t_res = timed(lambda: bc.join_residual(cl, cr, keep, n_left, n_right, leg))
        if rnd:
            times[leg]["candidate"].append(t_cand)
            times[leg]["filter"].append(t_filt)
            times[leg]["residual"].append(t_res)
        results[leg] = (len(ol), None if orr is None else orr.null_count, None if orr is None else len(orr))
        m = len(cl)
        del ol, orr, keep
        if rnd < args.reps:
            del cl, cr

# invariants on the last round's candidates, evaluated with torch
tl, tr = rows(cl), rows(cr)
passing = lv_valid[tl] & rw_valid[tr] & (lv[tl] < rw[tr])
n_pass = int(passing.sum())
left_with = int(torch.unique(tl[passing]).numel())
right_with = int(torch.unique(tr[passing]).numel())
anti = bc.join_residual(cl, cr, bc.less(bc.take(d_lv, cl), bc.take(d_rw, cr)), n_left, n_right, "left anti")[0]
left_outer_rows = n_pass + (n_left - left_with)
checks = {
    "inner": results["inner"][0] == n_pass,
    "left semi": results["left semi"][0] == left_with and results["left semi"][0] + len(anti) == n_left,
    "left outer": results["left outer"][0] == left_outer_rows and results["left outer"][1] == n_left - left_with,
    "full outer": results["full outer"][0] == left_outer_rows + (n_right - right_with),
}

gpu = torch.cuda.get_device_name(0)
try:
    import pynvml
    pynvml.nvmlInit()
    power = pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000
except Exception:
    power = None
keep_bits = 2 * ((m + 7) // 8)  # values + validity of the keep flags
for leg in LEGS:
    out_rows = results[leg][0]
    scans = {"inner": 0, "left semi": 1, "left outer": 2, "full outer": 2}[leg]
    reads = 8 * m + keep_bits + 4 * n_left * scans
    writes = 4 * out_rows if leg == "left semi" else 8 * out_rows + (out_rows + 7) // 8 * (2 if leg == "full outer" else
                                                                                          1 if leg == "left outer" else 0)
    med = {k: statistics.median(v) for k, v in times[leg].items()}
    print(json.dumps({"leg": leg, "probe_rows": n_left, "build_rows": n_right, "candidates": m, "passing": n_pass,
                      "result_rows": out_rows, "candidate_ms": round(med["candidate"], 3), "filter_ms": round(med["filter"], 3),
                      "residual_ms": round(med["residual"], 3),
                      "residual_min_max_ms": [round(min(times[leg]["residual"]), 3), round(max(times[leg]["residual"]), 3)],
                      "residual_alg_bytes": reads + writes,
                      "residual_share_of_3.35TBps": round((reads + writes) / (med["residual"] * 1e-3) / 3.35e12, 3),
                      "parity_ok": bool(checks[leg]), "gpu": gpu, "power_limit_w": power}), flush=True)
if not all(checks.values()):
    sys.exit(1)
