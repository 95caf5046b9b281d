"""Time the cumulative scans on the device with CUDA events, and a Cast float64 -> float32 in the same run as an anchor:
cumulative_sum int64 (skip_nulls), cumulative_sum_checked int64, cumulative_max float64 and cumulative_mean int64 ->
float64 over a column with nulls, and cumulative_sum float32 without nulls.  Each line gives the median time, the
algorithmic bytes per row (a scan reads and writes each value once: int64 with a nullable input and output reads
8.125 B/row and writes 8.125 B/row), that rate as a share of the H100 SXM data sheet's 3.35 TB/s, a parity flag (the
device against pyarrow.compute on a 1M-row prefix: a prefix of a scan is the scan of the prefix), and the card's name
and power limit read in the same run.  The float32 sum runs over quarter-integers so that its partial sums are exact
and the parity is bit for bit.

    python scripts/cumulative_bench.py --rows 1000000000 --null-p 0.1 --iters 10
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import pyarrow.compute as pc  # noqa: E402
import torch  # noqa: E402

import arrow_b200.compute as bc  # noqa: E402
from arrow_b200 import Context, DeviceArray  # noqa: E402

PEAK_GBS = 3350.0


def _gpu_info():
    return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()


def _validity(n, null_p, g):
    valid = torch.rand(n, device="cuda", generator=g) >= null_p
    bits = torch.zeros((n + 63) // 64 * 8 + 8, dtype=torch.uint8, device="cuda")
    full = n // 8 * 8
    bits[: n // 8] = (valid[:full].view(-1, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(1).to(torch.uint8)
    if n % 8:
        bits[n // 8] = sum(int(valid[full + k]) << k for k in range(n % 8))
    return valid, bits, int(n - valid.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--null-p", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    info = _gpu_info()  # fails without a GPU: there is nothing to measure then
    ctx = Context.get(0)
    n = args.rows
    g = torch.Generator(device="cuda").manual_seed(5)
    valid, bits, nulls = _validity(n, args.null_p, g)
    f64 = (torch.rand(n, device="cuda", dtype=torch.float64, generator=g) - 0.5) * 2e6
    small = torch.randint(-1000, 1000, (n,), device="cuda", dtype=torch.int64, generator=g)
    quarters = (torch.randint(-64, 64, (n,), device="cuda", dtype=torch.int32, generator=g).to(torch.float32) / 4)
    torch.cuda.synchronize()

    def dev(t, ty, nullable=True):
        if not nullable:
            return DeviceArray.from_pointers(ctx, ty, n, t.data_ptr(), keepalive=(t,))
        return DeviceArray.from_pointers(ctx, ty, n, t.data_ptr(), validity_ptr=bits.data_ptr(), null_count=nulls,
                                         keepalive=(t, bits))

    d64, di, dq = dev(f64, pa.float64()), dev(small, pa.int64()), dev(quarters, pa.float32(), False)
    # name: (call, pyarrow call on the prefix, bytes per row in + out, validity included)
    cases = {
        "cast float64 -> float32 (anchor)": (lambda: bc.cast(d64, pa.float32(), safe=False),
                                             lambda x: pc.cast(x["f64"], pa.float32(), safe=False), 12.25),
        "cumulative_sum int64 skip_nulls": (lambda: bc.cumulative_sum(di, skip_nulls=True),
                                            lambda x: pc.cumulative_sum(x["small"], skip_nulls=True), 16.25),
        "cumulative_sum_checked int64 skip_nulls": (lambda: bc.cumulative_sum_checked(di, skip_nulls=True),
                                                    lambda x: pc.cumulative_sum_checked(x["small"], skip_nulls=True), 16.25),
        "cumulative_max float64 skip_nulls": (lambda: bc.cumulative_max(d64, skip_nulls=True),
                                              lambda x: pc.cumulative_max(x["f64"], skip_nulls=True), 16.25),
        "cumulative_mean int64 -> float64 skip_nulls": (lambda: bc.cumulative_mean(di, skip_nulls=True),
                                                        lambda x: pc.cumulative_mean(x["small"], skip_nulls=True), 16.25),
        "cumulative_sum float32 no nulls": (lambda: bc.cumulative_sum(dq), lambda x: pc.cumulative_sum(x["q"]), 8.0),
    }
    m = min(n, 1 << 20)
    hmask = ~valid[:m].cpu().numpy()
    host = {"f64": pa.array(f64[:m].cpu().numpy(), mask=hmask), "small": pa.array(small[:m].cpu().numpy(), mask=hmask),
            "q": pa.array(quarters[:m].cpu().numpy())}
    stream = torch.cuda.ExternalStream(ctx.lib.b2_context_stream(ctx.handle))
    for name, (fn, ref, bpr) in cases.items():
        out = fn()
        parity = out.slice(0, m).to_arrow().equals(ref(host))
        del out
        ctx.sync()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(args.iters):
            start.record(stream)
            out = fn()
            end.record(stream)
            end.synchronize()
            times.append(start.elapsed_time(end))
            del out
        ms = float(np.median(times))
        gbs = bpr * n / ms / 1e6
        print(json.dumps({"case": name, "rows": n, "null_p": args.null_p, "median_ms": round(ms, 3), "bytes_per_row": round(bpr, 4),
                          "GB_per_s": round(gbs, 1), "share_of_3.35TBps": round(gbs / PEAK_GBS, 3), "parity": parity,
                          "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
