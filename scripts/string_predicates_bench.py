#!/usr/bin/env python
"""String predicates (csrc/string_predicates.cu) over the C5 column of bench_configs.py: `--rows` large_utf8 values of
0-32 random lowercase bytes with 10 % nulls.  Legs: equal and less against a scalar, equal array-array (the column
against a copy of itself, so every byte is read on both sides), starts_with / ends_with / match_substring with patterns
of 1, 3, 8 and 20 B, and a general match_like ("a%b_c%", one lane per row).  The C5 Filter of the same column (selectivity
0.5) is timed in the same run as a yardstick: it reads the same offsets and bytes and writes more.
Each leg is the median of `--reps` CUDA-event timings after one warm-up.  One JSON line per leg: the card and its power
limit, the algorithmic bytes (8 B of offsets + the row's bytes + 1/8 B of validity read, 2/8 B written per row; for
equal against a scalar only the bytes of rows of the scalar's length), their share of 3.35 TB/s, and a parity flag
(pyarrow.compute on three sampled 100k-row slices, and for equal / starts_with / ends_with of 1 and 3 B also a torch
count over the whole column)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyarrow as pa
import pyarrow.compute as pc
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=500_000_000)
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
n = args.rows
torch.cuda.set_device(0)
ctx = Context.get(0)
stream = torch.cuda.Stream()  # a stream of its own: the events must see the library's work
torch.cuda.set_stream(stream)
ctx.stream = stream.cuda_stream
gen = torch.Generator(device="cuda")
gen.manual_seed(0xC5)


def card_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return {"gpu": name, "power_limit_w": power}


def packed(mask: torch.Tensor) -> torch.Tensor:
    m = mask.numel()
    bits = torch.cat([mask, torch.zeros((-m) % 8 + 64, dtype=torch.bool, device="cuda")]).view(-1, 8).to(torch.uint8)
    weights = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device="cuda")
    return (bits * weights).sum(dim=1, dtype=torch.uint8)


def timed(fn):
    out, times = None, []
    for r in range(args.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        out = None
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        if r:
            times.append(e0.elapsed_time(e1))
    return statistics.median(times), out


card = card_info()
lens = torch.randint(0, 33, (n,), dtype=torch.int64, device="cuda", generator=gen)
offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
torch.cumsum(lens, 0, out=offs[1:])
total = int(offs[-1])
data = torch.randint(97, 123, (total + 64,), dtype=torch.uint8, device="cuda", generator=gen)
valid = torch.rand(n, device="cuda", generator=gen) >= 0.1
vbits = packed(valid)
torch.cuda.synchronize()
col = DeviceArray.from_pointers(ctx, pa.large_string(), n, offs.data_ptr(), validity_ptr=vbits.data_ptr(), null_count=-1,
                                data2_ptr=data.data_ptr(), keepalive=(offs, data, vbits))
L = total / n
per_row = 8 + L + 1 / 8 + 2 / 8


def torch_count(kind: str, pat: bytes) -> int:
    """true and valid rows of equal / starts_with / ends_with over the whole column, 64M rows at a time"""
    count = 0
    m = len(pat)
    p = torch.tensor(list(pat), dtype=torch.uint8, device="cuda")
    for s0 in range(0, n, 1 << 26):
        ln = lens[s0:s0 + (1 << 26)]
        o0, o1 = offs[s0:s0 + ln.numel()], offs[s0 + 1:s0 + 1 + ln.numel()]
        ok = (ln == m) if kind == "equal" else (ln >= m)
        base = o0 if kind != "ends_with" else o1 - m
        for k in range(m):
            ok &= data[(base + k).clamp(0, total - 1)] == p[k]
        count += int((ok & valid[s0:s0 + (1 << 26)]).sum())
    return count


def sampled_parity(out: DeviceArray, fn) -> bool:
    ok = True
    for s0 in (0, n // 2, n - 100_000):
        host = col.slice(s0, 100_000).to_arrow()
        ok = ok and out.slice(s0, 100_000).to_arrow().equals(fn(host))
    return ok


def report(leg, ms, alg, parity, extra=None):
    rec = {"leg": leg, "rows": n, "mean_len": round(L, 3), "ms": round(ms, 3), "alg_bytes": int(alg),
           "share_of_3.35TBps": round(alg / (ms * 1e-3) / 3.35e12, 3), "parity": bool(parity)}
    rec.update(extra or {})
    rec.update(card)
    print(json.dumps(rec), flush=True)


def true_count(out: DeviceArray) -> int:
    a = out.to_arrow()
    return int(pc.sum(pc.and_kleene(a, a.is_valid())).as_py() or 0)


# ---- filter yardstick (C5) -------------------------------------------------------------------------------------
mask_bits = packed(torch.rand(n, device="cuda", generator=gen) < 0.5)
mask = DeviceArray.from_pointers(ctx, pa.bool_(), n, mask_bits.data_ptr(), keepalive=mask_bits)
ms, out = timed(lambda: bc.filter(col, mask))
report("c5 filter large_utf8 s=0.5 (yardstick)", ms, n * (8 + L + 0.25) + 0.5 * n * (8 + L + 0.125), out.length > 0)
del out, mask, mask_bits
torch.cuda.empty_cache()

# ---- compares ----------------------------------------------------------------------------------------------------
sc = "abc"
ms, out = timed(lambda: bc.equal(col, sc))
same_len = int((lens == len(sc)).sum())
report("equal(s, 'abc')", ms, n * (8 + 1 / 8 + 2 / 8) + same_len * len(sc),
       sampled_parity(out, lambda h: pc.equal(h, sc)) and true_count(out) == torch_count("equal", sc.encode()))
ms, out = timed(lambda: bc.less(col, "m"))
report("less(s, 'm')", ms, n * per_row, sampled_parity(out, lambda h: pc.less(h, "m")))
data2 = data.clone()
col2 = DeviceArray.from_pointers(ctx, pa.large_string(), n, offs.data_ptr(), validity_ptr=vbits.data_ptr(), null_count=-1,
                                 data2_ptr=data2.data_ptr(), keepalive=(offs, data2, vbits))
ms, out = timed(lambda: bc.equal(col, col2))
report("equal(s, copy of s) array-array", ms, n * (2 * (8 + L + 1 / 8) + 2 / 8),
       sampled_parity(out, lambda h: pc.equal(h, h)) and true_count(out) == int(valid.sum()))
del col2, data2, out
torch.cuda.empty_cache()

# ---- matches -----------------------------------------------------------------------------------------------------
for pat in ("e", "abc", "abcdefgh", "qwertyuiopasdfghjklz"):
    for fn in ("starts_with", "ends_with", "match_substring"):
        ms, out = timed(lambda: getattr(bc, fn)(col, pat))
        ok = sampled_parity(out, lambda h: getattr(pc, fn)(h, pat))
        if fn != "match_substring" and len(pat) <= 3:
            ok = ok and true_count(out) == torch_count(fn, pat.encode())
        report(f"{fn}(s, {len(pat)} B)", ms, n * per_row, ok, {"pattern_bytes": len(pat)})
ms, out = timed(lambda: bc.match_like(col, "a%b_c%"))
report("match_like(s, 'a%b_c%') general matcher", ms, n * per_row, sampled_parity(out, lambda h: pc.match_like(h, "a%b_c%")))
