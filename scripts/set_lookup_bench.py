#!/usr/bin/env python
"""is_in / index_in (csrc/set_lookup.cu) over `--rows` int64 values with 10 % nulls, half of them drawn from the value set:
  is_in against 8 values (table in shared memory), against sets just below and above the shared-memory threshold, against
  1M values (global table, L2-resident) and 10M values (beyond L2); index_in against 1,000 values; is_in over
  `--strings` large_utf8 values of 0-32 bytes against 25 words.
Build (b2_set_lookup_create) and probe (b2_is_in / b2_index_in) are timed apart with CUDA events, median of `--reps` after
one warm-up.  Next to every numeric leg, compare(values, scalar) on the same column is timed as a yardstick: it moves the
same bytes per row as a small-set is_in.  One JSON line per leg: the card and its power limit, the algorithmic bytes
(int64 is_in reads 8 + 1/8 B and writes 1/8 B per row, + 1/8 B when the result has validity; index_in writes
4 + 1/8 B), their share of 3.35 TB/s, and a parity flag (torch.isin on the same data for numbers; a sampled pyarrow
check for strings)."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray, _cabi

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000_000)
ap.add_argument("--strings", type=int, default=500_000_000)
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
n = args.rows
torch.cuda.set_device(0)
ctx = Context.get(0)
stream = torch.cuda.Stream()  # a stream of its own: NULL would make the library use its own, which the events do not see
torch.cuda.set_stream(stream)
ctx.stream = stream.cuda_stream
lib = ctx.lib
gen = torch.Generator(device="cuda")
gen.manual_seed(0x5E7)


def packed_validity(m: int, null_p: float):
    """(LSB-first validity bitmap, bool mask) with about null_p nulls"""
    valid = torch.rand(m, device="cuda", generator=gen) >= null_p
    pad = (-m) % 8
    bits = torch.cat([valid, torch.zeros(pad, dtype=torch.bool, device="cuda")]).view(-1, 8).to(torch.uint8)
    weights = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device="cuda")
    return (bits * weights).sum(dim=1, dtype=torch.uint8), valid


def timed(fn, reps):
    out, times = None, []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        out = None
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        if r:
            times.append(e0.elapsed_time(e1))
    return statistics.median(times), out


def count_true(arr: DeviceArray) -> int:
    c, cnt = arr._c(), C.c_int64()
    if c.validity:  # true and valid
        tmp = ctx.alloc((arr.length + 7) // 8 + 16)
        assert lib.b2_bitmap_and(ctx.handle, c.data, 0, c.validity, 0, arr.length, tmp.ptr, C.byref(cnt), ctx.stream) == 0
        return cnt.value
    assert lib.b2_bitmap_count(ctx.handle, c.data, 0, arr.length, C.byref(cnt), ctx.stream) == 0
    return cnt.value


def leg(name, values: DeviceArray, value_set: DeviceArray, function: str, behavior: str, bytes_per_row_in: float,
        parity_fn, yardstick=None):
    cvs, h = value_set._c(), C.c_void_p()
    nm = bc.NULL_MATCHING[behavior]

    def build():
        assert lib.b2_set_lookup_create(ctx.handle, C.byref(cvs), nm, C.byref(h), ctx.stream) == 0, _cabi.last_error()
        return h
    build_times = []
    for r in range(args.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        build()
        e1.record()
        e1.synchronize()
        if r:
            build_times.append(e0.elapsed_time(e1))
        if r < args.reps:
            lib.b2_set_lookup_destroy(h)
    nbytes, shared = C.c_int64(), C.c_int32()
    lib.b2_set_lookup_table(h, C.byref(nbytes), C.byref(shared))
    probe = getattr(lib, "b2_" + function)
    cv = values._c()

    def run():
        co = _cabi.B2Array()
        assert probe(h, C.byref(cv), C.byref(co), ctx.stream) == 0, _cabi.last_error()
        return bc._out(ctx, co, pa.int32() if function == "index_in" else pa.bool_())
    ms, out = timed(run, args.reps)
    lib.b2_set_lookup_destroy(h)
    rows = values.length
    has_valid = out._c().validity is not None
    out_bytes = (4 if function == "index_in" else 0) + 1 / 8 + (1 / 8 if has_valid or function == "index_in" else 0)
    alg = rows * (bytes_per_row_in + out_bytes)
    rec = {"leg": name, "function": function, "behavior": behavior, "rows": rows, "set_size": value_set.length,
           "table_bytes": nbytes.value, "table_in_shared_memory": bool(shared.value),
           "build_ms": round(statistics.median(build_times), 3), "probe_ms": round(ms, 3), "alg_bytes": int(alg),
           "share_of_3.35TBps": round(alg / (ms * 1e-3) / 3.35e12, 3), "parity": bool(parity_fn(out))}
    if yardstick is not None:
        yms, _ = timed(yardstick, args.reps)
        rec["compare_scalar_ms"] = round(yms, 3)
    rec.update(card)
    print(json.dumps(rec), flush=True)


def card_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(q.splitlines()[0])
    except Exception:
        power = None
    return {"gpu": name, "power_limit_w": power}


card = card_info()

# ---- int64 legs ------------------------------------------------------------------------------------------------
vbits, vmask = packed_validity(n, 0.10)
raw = torch.randint(-(1 << 40), 1 << 40, (n,), dtype=torch.int64, device="cuda", generator=gen)
hit = torch.rand(n, device="cuda", generator=gen) < 0.5
values_t = torch.empty_like(raw)
dv = DeviceArray.from_pointers(ctx, pa.int64(), n, values_t.data_ptr(), validity_ptr=vbits.data_ptr(), null_count=-1,
                               keepalive=(values_t, vbits))
probe_bytes = 8 + 1 / 8  # values + validity


def numeric_leg(name, m, function="is_in", behavior="match"):
    set_t = torch.randint(-(1 << 40), 1 << 40, (m,), dtype=torch.int64, device="cuda", generator=gen)
    pick = torch.randint(0, m, (n,), device="cuda", generator=gen)
    torch.where(hit, set_t[pick], raw, out=values_t)
    del pick
    torch.cuda.synchronize()
    dset = DeviceArray.from_pointers(ctx, pa.int64(), m, set_t.data_ptr(), keepalive=set_t)

    def parity(out):
        want = int((torch.isin(values_t, set_t) & vmask).sum())
        if function == "index_in":
            return out.null_count == n - want
        return count_true(out) == want
    leg(name, dv, dset, function, behavior, probe_bytes, parity, yardstick=lambda: bc.equal(dv, pa.scalar(5, pa.int64())))


def stages_in_shared_memory(m: int) -> bool:
    t = torch.arange(m, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return bc.set_lookup_table(DeviceArray.from_pointers(ctx, pa.int64(), m, t.data_ptr(), keepalive=t))[1]


below = 1  # the most distinct values the shared-memory placement takes (a power of two)
while stages_in_shared_memory(2 * below):
    below *= 2
numeric_leg("is_in int64, 8 values (shared memory)", 8)
numeric_leg(f"is_in int64, {below} values (just below the shared-memory threshold)", below)
numeric_leg(f"is_in int64, {below + 1} values (just above: global memory)", below + 1)
numeric_leg("is_in int64, 1M values (global, L2-resident)", 1 << 20)
numeric_leg("is_in int64, 10M values (global, beyond L2)", 10_000_000)
numeric_leg("index_in int64, 1000 values", 1000, function="index_in")
numeric_leg("is_in int64, 8 values, inconclusive", 8, behavior="inconclusive")
del dv, values_t, raw, hit, vbits, vmask
torch.cuda.empty_cache()

# ---- large_utf8 leg ----------------------------------------------------------------------------------------------
ns = args.strings
vocab_n = 1000
rng = np.random.default_rng(1)
vocab = ["".join(chr(97 + c) for c in rng.integers(0, 26, L)) for L in rng.integers(0, 33, vocab_n)]
vocab = list(dict.fromkeys(vocab))
vocab_n = len(vocab)
pad = torch.zeros((vocab_n, 32), dtype=torch.uint8)
for i, w in enumerate(vocab):
    pad[i, :len(w)] = torch.tensor(list(w.encode()), dtype=torch.uint8) if w else pad[i, :0]
pad = pad.cuda()
lens = torch.tensor([len(w) for w in vocab], dtype=torch.int64, device="cuda")
ids = torch.randint(0, vocab_n, (ns,), device="cuda", generator=gen)
offsets = torch.zeros(ns + 1, dtype=torch.int64, device="cuda")
torch.cumsum(lens[ids], 0, out=offsets[1:])
total = int(offsets[-1])
chars = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
step = 50_000_000
pos = torch.arange(32, device="cuda")
for s0 in range(0, ns, step):
    cid = ids[s0:s0 + step]
    sel = pad[cid].masked_select(pos[None, :] < lens[cid][:, None])
    chars[int(offsets[s0]):int(offsets[s0]) + sel.numel()] = sel
    del sel
sbits, _ = packed_validity(ns, 0.10)
torch.cuda.synchronize()
dstr = DeviceArray.from_pointers(ctx, pa.large_string(), ns, offsets.data_ptr(), validity_ptr=sbits.data_ptr(), null_count=-1,
                                 data2_ptr=chars.data_ptr(), keepalive=(offsets, chars, sbits))
words = pa.array(vocab[:25], pa.large_string())
dwords = DeviceArray.from_arrow(words, ctx)


def string_parity(out):
    ok = True
    for s0 in (0, ns // 2, ns - 100_000):
        host = dstr.slice(s0, 100_000).to_arrow()
        ok = ok and out.slice(s0, 100_000).to_arrow().equals(pc.is_in(host, value_set=words))
    return ok


leg("is_in large_utf8 0-32 B, 25 words", dstr, dwords, "is_in", "match", 8 + 1 / 8 + total / ns, string_parity)
