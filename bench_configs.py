#!/usr/bin/env python
"""bench_configs.py -- the other BASELINE.json configs at scale (not the driver's bench line):
  c1  Filter(int64, bool mask)            1B rows, values null_p 0.1, mask non-null, s = 0.5
  c3  group-by sum+count, int64 key/value 1B rows, 10M groups (fused table and Grouper+aggregators)
  c3u group-by / dictionary_encode with a large_utf8 key   500M strings from 1M distinct words (not in the default --only list)
  join inner hash join: n/2 probe rows against 10M unique build keys (not in the default --only list)
  c4  SortIndices int64 + validity        1B rows (wide range) and narrow range [0, 4095]
  c4s SortIndices large_utf8 + validity   500M words (1M distinct, 8-16 B) and 500M random 0-32 B strings (not in the
      default --only list); each line carries a parity_ok flag computed in the same run
  f1  dictionary_encode / value_counts of an int64 column (1M distinct values), 500M rows
  c5  large_utf8 Filter                   500M strings, 0-32 B, null_p 0.1, s = 0.5  (+ dictionary Take)
  cmp compare int64 -> bool               1B rows
Each prints one JSON line: rows/s, algorithmic GB/s (SURVEY.md section 8d byte model) and the
fraction of the measured copy peak.  Inputs are generated on the device with torch (plumbing).
Usage: python bench_configs.py [--rows N] [--only c1,c3,...] [--reps K]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import pyarrow as pa
import torch

import arrow_b200.compute as bc
from arrow_b200 import Context, DeviceArray
from bench import NULL_P, SEED, make_validity, measured_peaks


def timed(stream, fn, reps, warmup=2):
    for _ in range(warmup):
        r = fn()
        del r
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(reps):
        r = fn()
        del r
    b.record(stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


class _Cai:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def _cai(ptr, n, typestr):
    return _Cai(ptr, n, typestr)


def report(name, n, ms, alg_bytes, extra=None):
    peak, _ = measured_peaks()
    gbs = alg_bytes / (ms * 1e-3) / 1e9
    line = {"config": name, "rows": n, "ms": ms, "rows_per_s": n / (ms * 1e-3), "alg_bytes": alg_bytes, "gbs": gbs,
            "frac_of_measured_peak": gbs / peak}
    if extra:
        line.update(extra)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--only", default="c1,cmp,c3,c4,c5,f1")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fused-only", action="store_true", help="c3: stop after the fused group-by")
    ap.add_argument("--groups", type=int, default=0, help="c3: number of distinct keys (default 10M at >= 100M rows)")
    args = ap.parse_args()
    only = set(args.only.split(","))
    n = args.rows
    torch.cuda.set_device(0)
    ctx = Context.get(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.stream = stream.cuda_stream
    gen = torch.Generator(device="cuda")
    gen.manual_seed(SEED)

    if "c1" in only or "cmp" in only:
        vals_t = torch.randint(-100, 101, (n,), dtype=torch.int64, device="cuda", generator=gen)
        vvalid_t, v_nulls = make_validity(torch, n, gen)
        values = DeviceArray.from_pointers(ctx, pa.int64(), n, vals_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)
        if "c1" in only:
            for sel in (0.5, 0.01, 0.999):
                m8 = (n + 7) // 8 * 8
                mask_bits = torch.empty(m8 // 8 + 64, dtype=torch.uint8, device="cuda")
                from bench import pack_bits
                chunk = 1 << 27
                for lo in range(0, m8, chunk):
                    m = min(chunk, m8 - lo)
                    mask_bits[lo // 8:(lo + m) // 8] = pack_bits(torch, torch.rand(m, device="cuda", generator=gen) < sel)
                mask = DeviceArray.from_pointers(ctx, pa.bool_(), n, mask_bits.data_ptr())
                ms = timed(stream, lambda: bc.filter(values, mask), args.reps)
                out_len = len(bc.filter(values, mask))
                s = out_len / n
                report(f"c1 filter int64 sel={sel}", n, ms, n * (8 + 0.125 + 0.125) + out_len * 8.125, {"selectivity": s})
                del mask, mask_bits
        if "cmp" in only:
            other_t = torch.randint(-100, 101, (n,), dtype=torch.int64, device="cuda", generator=gen)
            other = DeviceArray.from_pointers(ctx, pa.int64(), n, other_t.data_ptr())
            ms = timed(stream, lambda: bc.greater(values, other), args.reps)
            report("compare greater(int64,int64)", n, ms, n * (16 + 0.125 + 0.25))
            ms = timed(stream, lambda: bc.sum(values), args.reps)
            report("f2 sum/mean/min_max state of int64 (b2_reduce)", n, ms, n * (8 + 0.125))
            del other, other_t
        del values, vals_t, vvalid_t

    if "c3" in only:
        groups = args.groups or (10_000_000 if n >= 100_000_000 else max(1000, n // 100))
        keys_t = torch.randint(0, groups, (n,), dtype=torch.int64, device="cuda", generator=gen)
        vals_t = torch.randint(-100, 101, (n,), dtype=torch.int64, device="cuda", generator=gen)
        vvalid_t, v_nulls = make_validity(torch, n, gen)
        keys = DeviceArray.from_pointers(ctx, pa.int64(), n, keys_t.data_ptr())
        vals = DeviceArray.from_pointers(ctx, pa.int64(), n, vals_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)

        paths = {}

        def fused():
            g = bc.GroupBySumCount(pa.int64(), pa.int64(), expected_groups=groups, ctx=ctx)
            g.consume(keys, vals)
            paths["counts"] = g.path_counts()
            return g.finalize()
        ms = timed(stream, fused, args.reps, warmup=1)
        ng = len(fused()[0])
        report("c3 group-by sum+count (fused table)", n, ms, n * 16.125 + ng * 24.25,
               {"groups": ng, "paths": paths["counts"]})
        if args.fused_only:
            return

        def unfused():
            return bc.group_by([keys], [("hash_sum", vals, None), ("hash_count", vals, None)], fused=False)
        ms = timed(stream, unfused, max(1, args.reps - 1), warmup=1)
        report("c3 group-by sum+count (Grouper + 2 HashAggregators)", n, ms, n * 16.125 + ng * 24.25, {"groups": ng})
        del keys, vals, keys_t, vals_t, vvalid_t

    if "c3u" in only:
        # group-by with a large_utf8 key: n/2 strings from 1M distinct words of 8-16 B (bench.make_word_column)
        from bench import make_word_column
        m = n // 2
        vocab = 1_000_000 if m >= 10_000_000 else max(100, m // 100)
        kid, offs, data, total = make_word_column(torch, gen, m, vocab)
        vals_t = torch.randint(-100, 101, (m,), dtype=torch.int64, device="cuda", generator=gen)
        vvalid_t, v_nulls = make_validity(torch, m, gen)
        skeys = DeviceArray.from_pointers(ctx, pa.large_string(), m, offs.data_ptr(), data2_ptr=data.data_ptr())
        vals = DeviceArray.from_pointers(ctx, pa.int64(), m, vals_t.data_ptr(), validity_ptr=vvalid_t.data_ptr(), null_count=v_nulls)
        ms = timed(stream, lambda: bc.group_by([skeys], [("hash_sum", vals, None), ("hash_count", vals, None)], fused=False),
                   max(1, args.reps - 1), warmup=1)
        L = total / m
        report("c3u group-by sum+count, large_utf8 key (1M distinct words)", m, ms, m * (8 + L + 8.125) + vocab * (8 + L + 16.25),
               {"groups": vocab, "mean_len": L})
        ms = timed(stream, lambda: bc.dictionary_encode(skeys), max(1, args.reps - 1), warmup=1)
        report("f1 dictionary_encode large_utf8 (1M distinct words)", m, ms, m * (8 + L + 4) + vocab * (8 + L), {"mean_len": L})
        del skeys, vals, kid, offs, data, vals_t, vvalid_t

    if "join" in only:
        # inner hash join: n/2 probe rows (int64 keys, uniform over 1.25x the build keys, so 80 % match) against 10M unique build keys
        m = n // 2
        nb = 10_000_000 if m >= 100_000_000 else max(1000, m // 50)
        build_t = torch.randperm(int(nb * 1.25), device="cuda", generator=gen)[:nb].to(torch.int64)
        probe_t = torch.randint(0, int(nb * 1.25), (m,), dtype=torch.int64, device="cuda", generator=gen)
        build = DeviceArray.from_pointers(ctx, pa.int64(), nb, build_t.data_ptr())
        probe = DeviceArray.from_pointers(ctx, pa.int64(), m, probe_t.data_ptr())
        ms = timed(stream, lambda: bc.hash_join_indices([probe], [build], "inner"), max(1, args.reps - 1), warmup=1)
        li, ri = bc.hash_join_indices([probe], [build], "inner")
        pairs = len(li)
        # parity: every emitted pair has equal keys, and the pair count equals the number of probe keys present in the build side
        lt = torch.as_tensor(_cai(li.buffers[1].ptr, pairs, "<u4"), device="cuda").to(torch.int64)
        rt = torch.as_tensor(_cai(ri.buffers[1].ptr, pairs, "<u4"), device="cuda").to(torch.int64)
        present = torch.zeros(int(nb * 1.25), dtype=torch.bool, device="cuda")
        present[build_t] = True
        ok = bool((probe_t[lt] == build_t[rt]).all().item()) and pairs == int(present[probe_t].sum().item())
        report("join inner: 10M unique int64 build keys, probe keys 80 % matching", m, ms, m * 8 + nb * 8 + pairs * 8,
               {"build_rows": nb, "pairs": pairs, "parity_ok": ok})
        del build, probe, build_t, probe_t, li, ri, lt, rt, present

    if "c4" in only:
        m = min(n, (1 << 30) - 1)
        for name, lo, hi in (("wide [-2^62,2^62)", -2**62, 2**62), ("narrow [0,4095]", 0, 4096)):
            keys_t = torch.randint(lo, hi, (m,), dtype=torch.int64, device="cuda", generator=gen)
            kvalid_t, k_nulls = make_validity(torch, m, gen)
            keys = DeviceArray.from_pointers(ctx, pa.int64(), m, keys_t.data_ptr(), validity_ptr=kvalid_t.data_ptr(), null_count=k_nulls)
            ms = timed(stream, lambda: bc.array_sort_indices(keys), max(1, args.reps - 1), warmup=1)
            report(f"c4 sort_indices int64 {name}", m, ms, m * 16.125)
            del keys, keys_t, kvalid_t
            ctx.trim()

    if "c4s" in only:
        from bench import make_word_column, unpack_bits
        m = n // 2
        # (a) the word column of c3u: the first five letters are the base-26 digits of the word id, the rest depends on
        # the id only, so the expected order is a stable sort of the ids with the nulls moved to the end
        vocab = 1_000_000 if m >= 10_000_000 else max(100, m // 100)
        kid, offs, data, total = make_word_column(torch, gen, m, vocab)
        svalid_t, s_nulls = make_validity(torch, m, gen)
        words = DeviceArray.from_pointers(ctx, pa.large_string(), m, offs.data_ptr(), validity_ptr=svalid_t.data_ptr(),
                                          null_count=s_nulls, data2_ptr=data.data_ptr())
        ms = timed(stream, lambda: bc.array_sort_indices(words), max(1, args.reps - 1), warmup=1)
        got = bc.array_sort_indices(words)
        ctx.sync()
        ctx.trim()
        got_t = torch.as_tensor(_cai(got.buffers[1].ptr, m, "<i8"), device="cuda")
        valid = unpack_bits(torch, svalid_t, m)
        ok = bool(torch.equal(got_t, torch.sort(torch.where(valid, kid, vocab), stable=True).indices))
        L = total / m
        report("c4s sort_indices large_utf8 words (1M distinct, 8-16 B)", m, ms, m * (8 + L + 0.125 + 8),
               {"mean_len": L, "distinct": vocab, "parity_ok": ok})
        del words, got, got_t, valid, kid, offs, data, svalid_t
        ctx.trim()
        torch.cuda.empty_cache()
        # (b) the random 0-32 B lowercase strings of c5.  No zero byte occurs, so the zero-padded 32 bytes read as four
        # big-endian int64 words order exactly like the strings: four stable sorts, least significant word first
        lens = torch.randint(0, 33, (m,), dtype=torch.int64, device="cuda", generator=gen)
        offs = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens, 0, out=offs[1:])
        total = int(offs[-1].item())
        data = torch.randint(97, 123, (total + 64,), dtype=torch.uint8, device="cuda", generator=gen)
        svalid_t, s_nulls = make_validity(torch, m, gen)
        strs = DeviceArray.from_pointers(ctx, pa.large_string(), m, offs.data_ptr(), validity_ptr=svalid_t.data_ptr(), null_count=s_nulls,
                                         data2_ptr=data.data_ptr())
        ms = timed(stream, lambda: bc.array_sort_indices(strs), max(1, args.reps - 1), warmup=1)
        got = bc.array_sort_indices(strs)
        ctx.sync()
        ctx.trim()
        got_t = torch.as_tensor(_cai(got.buffers[1].ptr, m, "<i8"), device="cuda")
        words4 = torch.empty((4, m), dtype=torch.int64, device="cuda")
        col = torch.arange(32, device="cuda", dtype=torch.int64)
        shifts = torch.arange(56, -8, -8, device="cuda", dtype=torch.int64)
        for lo in range(0, m, 1 << 22):
            hi = min(m, lo + (1 << 22))
            b = data[(offs[lo:hi, None] + col).clamp(max=total + 63)].to(torch.int64)
            b = torch.where(col < lens[lo:hi, None], b, 0).view(hi - lo, 4, 8)
            words4[:, lo:hi] = (b << shifts).sum(-1).T
            del b
        perm = torch.arange(m, device="cuda", dtype=torch.int64)
        for w in (3, 2, 1, 0):
            perm = perm[torch.sort(words4[w][perm], stable=True).indices]
        valid = unpack_bits(torch, svalid_t, m)
        perm = torch.cat([perm[valid[perm]], torch.nonzero(~valid).flatten()])  # nulls after the strings, in row order
        ok = bool(torch.equal(got_t, perm))
        L = total / m
        report("c4s sort_indices large_utf8 random 0-32 B", m, ms, m * (8 + L + 0.125 + 8), {"mean_len": L, "parity_ok": ok})
        del strs, got, got_t, words4, perm, valid, lens, offs, data, svalid_t
        ctx.trim()
        torch.cuda.empty_cache()

    if "c5" in only:
        m = n // 2
        lens = torch.randint(0, 33, (m,), dtype=torch.int64, device="cuda", generator=gen)
        offs = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
        torch.cumsum(lens, 0, out=offs[1:])
        total = int(offs[-1].item())
        del lens
        data = torch.randint(97, 123, (total + 64,), dtype=torch.uint8, device="cuda", generator=gen)
        svalid_t, s_nulls = make_validity(torch, m, gen)
        strs = DeviceArray.from_pointers(ctx, pa.large_string(), m, offs.data_ptr(), validity_ptr=svalid_t.data_ptr(), null_count=s_nulls,
                                         data2_ptr=data.data_ptr())
        from bench import pack_bits
        m8 = (m + 7) // 8 * 8
        mask_bits = torch.empty(m8 // 8 + 64, dtype=torch.uint8, device="cuda")
        chunk = 1 << 27
        for lo in range(0, m8, chunk):
            c = min(chunk, m8 - lo)
            mask_bits[lo // 8:(lo + c) // 8] = pack_bits(torch, torch.rand(c, device="cuda", generator=gen) < 0.5)
        mask = DeviceArray.from_pointers(ctx, pa.bool_(), m, mask_bits.data_ptr())
        ms = timed(stream, lambda: bc.filter(strs, mask), args.reps, warmup=1)
        L = total / m
        report("c5 filter large_utf8 s=0.5", m, ms, m * (8 + L + 0.25) + 0.5 * m * (8 + L + 0.125), {"mean_len": L})
        del strs, offs, data, svalid_t, mask, mask_bits
        # dictionary-encoded Take: int32 index column, int64 take-indices
        dict_idx_t = torch.randint(0, 1_000_000, (m,), dtype=torch.int32, device="cuda", generator=gen)
        col = DeviceArray.from_pointers(ctx, pa.int32(), m, dict_idx_t.data_ptr())
        take_idx_t = torch.randint(0, m, (m,), dtype=torch.int64, device="cuda", generator=gen)
        take_idx = DeviceArray.from_pointers(ctx, pa.int64(), m, take_idx_t.data_ptr())
        ms = timed(stream, lambda: bc.take(col, take_idx), args.reps, warmup=1)
        report("c5 dictionary take (int32 index column, random int64 idx)", m, ms, m * (8 + 4 + 4))
        del col, take_idx, dict_idx_t, take_idx_t

    if "f1" in only:
        # SURVEY 8f rank 1: produce config 5's dictionary column on the device
        m = n // 2
        distinct = 1_000_000
        keys_t = torch.randint(0, distinct, (m,), dtype=torch.int64, device="cuda", generator=gen)
        kvalid_t, k_nulls = make_validity(torch, m, gen)
        col = DeviceArray.from_pointers(ctx, pa.int64(), m, keys_t.data_ptr(), validity_ptr=kvalid_t.data_ptr(), null_count=k_nulls)
        ms = timed(stream, lambda: bc.dictionary_encode(col), args.reps, warmup=1)
        nd = len(bc.unique(col))
        report("f1 dictionary_encode int64 (1M distinct, null_p 0.1)", m, ms, m * (8 + 0.125 + 4 + 0.125) + nd * 8, {"dictionary": nd})
        ms = timed(stream, lambda: bc.value_counts(col), args.reps, warmup=1)
        report("f1 value_counts int64 (1M distinct, null_p 0.1)", m, ms, m * (8 + 0.125) + nd * 16, {"dictionary": nd})


if __name__ == "__main__":
    main()
