#!/usr/bin/env python
"""String transforms (csrc/string_transform.cu) over the C5 column of bench_configs.py: `--rows` large_utf8 values of
0-32 random lowercase bytes with 10 % nulls, and a second column of the same row lengths in which about a quarter of
the characters are two-byte (a 2-byte code point replaces two ASCII bytes), for the utf8 legs.
Legs: binary_length, utf8_length (2-byte column), ascii_upper, utf8_slice_codeunits(0, 8) and utf8_slice_codeunits(-4)
(2-byte column), binary_slice(2, 10) on a large_binary view of the C5 buffers, and binary_join_element_wise(s, s2, "-").
The C5 Filter (selectivity 0.5) is timed in the same run as a yardstick.
Each leg is the median of `--reps` CUDA-event timings after one warm-up.  One JSON line per leg: the card and its power
limit, the algorithmic bytes and their share of 3.35 TB/s, and a parity flag.  Algorithmic bytes per call:
  read : the input's offsets (8 B per row) and validity (1/8 B per row), plus the character bytes the function needs:
         none for binary_length and binary_slice's arithmetic, each row's bytes for utf8_length, ascii_upper and the
         utf8 slices (the walk may stop earlier; counted in full), the sliced bytes for binary_slice, both inputs' bytes
         (and offsets and validity) for the join;
  write: the output's validity (1/8 B per row), its offsets or values (8 B per row) and its character bytes.
Parity: pyarrow.compute on three sampled 100k-row slices for every leg; for binary_length, utf8_length and ascii_upper
also a torch restatement over the whole column, compared on the device row by row (equal(...) against it)."""
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
CHUNK = 1 << 26


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
n_valid = int(valid.sum())
# the 2-byte column: byte pairs (j, j + 1) at even j inside one row become U+00C0..U+00FF with probability 0.4, so a
# quarter of its characters are two-byte
data2 = data.clone()
row_start = torch.zeros(total + 1, dtype=torch.bool, device="cuda")
row_start[offs[:-1][lens > 0]] = True
for b0 in range(0, total - 1, 2 * CHUNK):
    j = torch.arange(b0, min(b0 + 2 * CHUNK, total - 1), 2, device="cuda")
    pick = j[(~row_start[j + 1]) & (torch.rand(j.numel(), device="cuda", generator=gen) < 0.4)]
    data2[pick] = 0xC3
    data2[pick + 1] = 0x80 + torch.randint(0, 64, (pick.numel(),), dtype=torch.uint8, device="cuda", generator=gen)
del row_start
torch.cuda.synchronize()


def column(buf, type_=pa.large_string()):
    return DeviceArray.from_pointers(ctx, type_, n, offs.data_ptr(), validity_ptr=vbits.data_ptr(), null_count=-1,
                                     data2_ptr=buf.data_ptr(), keepalive=(offs, buf, vbits))


col, col2, colb = column(data), column(data2), column(data, pa.large_binary())
L = total / n
vrow = 8 + 1 / 8  # offsets or values, and validity, per row


def sampled_parity(out: DeviceArray, src: DeviceArray, fn) -> bool:
    ok = True
    for s0 in (0, n // 2, n - 100_000):
        ok = ok and out.slice(s0, 100_000).to_arrow().equals(fn(src.slice(s0, 100_000).to_arrow()))
    return ok


def rows_equal(out: DeviceArray, want: DeviceArray) -> bool:
    """every valid row of out equals want's, compared on the device"""
    a = bc.equal(out, want).to_arrow()
    return int(pc.sum(pc.and_kleene(a, a.is_valid())).as_py() or 0) == n_valid


def report(leg, ms, alg, parity, extra=None):
    rec = {"leg": leg, "rows": n, "mean_len": round(L, 3), "ms": round(ms, 3), "alg_bytes": int(alg),
           "share_of_3.35TBps": round(alg / (ms * 1e-3) / 3.35e12, 3), "parity": bool(parity)}
    rec.update(extra or {})
    rec.update(card)
    print(json.dumps(rec), flush=True)


def out_bytes(out: DeviceArray) -> int:
    return int(bc.sum(bc.binary_length(out)).as_py() or 0)


# ---- filter yardstick (C5) -------------------------------------------------------------------------------------
mask_bits = packed(torch.rand(n, device="cuda", generator=gen) < 0.5)
mask = DeviceArray.from_pointers(ctx, pa.bool_(), n, mask_bits.data_ptr(), keepalive=mask_bits)
ms, out = timed(lambda: bc.filter(col, mask))
report("c5 filter large_utf8 s=0.5 (yardstick)", ms, n * (8 + L + 0.25) + 0.5 * n * (8 + L + 0.125), out.length > 0)
del out, mask, mask_bits
torch.cuda.empty_cache()

# ---- lengths -----------------------------------------------------------------------------------------------------
ms, out = timed(lambda: bc.binary_length(col))
want = DeviceArray.from_pointers(ctx, pa.int64(), n, lens.data_ptr(), keepalive=lens)
report("binary_length", ms, n * (vrow + vrow), sampled_parity(out, col, pc.binary_length) and rows_equal(out, want))
del out
lead = torch.zeros(n, dtype=torch.int64, device="cuda")  # torch restatement: bytes that are not 10xxxxxx, per row
for s0 in range(0, n, CHUNK):
    s1 = min(s0 + CHUNK, n)
    a, b = int(offs[s0]), int(offs[s1])
    rows = torch.repeat_interleave(torch.arange(s0, s1, device="cuda"), lens[s0:s1])
    lead.index_add_(0, rows, ((data2[a:b] & 0xC0) != 0x80).to(torch.int64))
    del rows
ms, out = timed(lambda: bc.utf8_length(col2))
want = DeviceArray.from_pointers(ctx, pa.int64(), n, lead.data_ptr(), keepalive=lead)
chars = int(lead.sum())
report("utf8_length (2-byte column)", ms, n * (vrow + vrow) + total, sampled_parity(out, col2, pc.utf8_length) and rows_equal(out, want),
       {"two_byte_share_of_chars": round((total - chars) / chars, 3)})
del out, want, lead
torch.cuda.empty_cache()

# ---- ascii_upper -------------------------------------------------------------------------------------------------
ms, out = timed(lambda: bc.ascii_upper(col))
upper = data - 32  # every byte of the column is a..z
want = column(upper)
report("ascii_upper", ms, n * (vrow + vrow) + 2 * total, sampled_parity(out, col, pc.ascii_upper) and rows_equal(out, want))
del out, want, upper
torch.cuda.empty_cache()

# ---- slices ------------------------------------------------------------------------------------------------------
for leg, start, stop in (("utf8_slice_codeunits(0, 8) (2-byte column)", 0, 8), ("utf8_slice_codeunits(-4) (2-byte column)", -4, None)):
    ms, out = timed(lambda: bc.utf8_slice_codeunits(col2, start, stop))
    ok = sampled_parity(out, col2, lambda h: pc.utf8_slice_codeunits(h, start, stop if stop is not None else (1 << 63) - 1))
    report(leg, ms, n * (vrow + vrow) + total + out_bytes(out), ok)
    del out
    torch.cuda.empty_cache()
ms, out = timed(lambda: bc.binary_slice(colb, 2, 10))
nb = out_bytes(out)
report("binary_slice(2, 10) (large_binary view)", ms, n * (vrow + vrow) + 2 * nb,
       sampled_parity(out, colb, lambda h: pc.binary_slice(h, 2, 10)))
del out
torch.cuda.empty_cache()

# ---- join --------------------------------------------------------------------------------------------------------
sep = pa.scalar("-", pa.large_string())
ms, out = timed(lambda: bc.binary_join_element_wise(col, col2, sep))
nb = out_bytes(out)


def join_ref(h):
    return pc.binary_join_element_wise(h, col2.slice(join_ref.s0, 100_000).to_arrow(), sep)


ok = True
for s0 in (0, n // 2, n - 100_000):
    join_ref.s0 = s0
    ok = ok and out.slice(s0, 100_000).to_arrow().equals(join_ref(col.slice(s0, 100_000).to_arrow()))
report("binary_join_element_wise(s, s2, '-')", ms, n * (2 * vrow + vrow) + 2 * total + nb, ok)
