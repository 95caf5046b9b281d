"""Time year / hour / subsecond over timestamp[us] and the casts timestamp[us] -> date32 and timestamp[ns] ->
timestamp[us] (safe) on the device, with CUDA events.  Each result carries a parity flag (the device against
pyarrow.compute on a 1M-row prefix) and the algorithmic bytes per row: 8 in + 8 out + 2/8 of validity (in and out)
for an int64 field, 16.25 B/row.

    python scripts/temporal_bench.py --rows 1000000000 --null-p 0.1 --iters 10
"""
import argparse
import ctypes as C
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
from arrow_b200 import Context, DeviceArray, _cabi  # noqa: E402


def _gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def _cast(ctx, dv, src, dst, truncate=False):
    cin, cout = dv._c(), _cabi.B2Array()
    f, t = bc.temporal_type(src), bc.temporal_type(dst)
    st = ctx.lib.b2_cast_temporal(ctx.handle, C.byref(cin), C.byref(f), C.byref(t), int(truncate), 0, C.byref(cout),
                                  ctx.stream)
    if st != 0:
        raise RuntimeError(_cabi.last_error())
    return DeviceArray._from_c(ctx, cout, dst)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 30)
    ap.add_argument("--null-p", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    ctx = Context.get(0)
    n = args.rows
    g = torch.Generator(device="cuda").manual_seed(1)
    # 1900 .. 2100 in microseconds; multiples of 1000 so that the safe ns -> us cast never fails
    lo, hi = -2208988800 * 10 ** 6, 4102444800 * 10 ** 6
    us = torch.randint(lo, hi, (n,), dtype=torch.int64, device="cuda", generator=g)
    valid = torch.rand(n, device="cuda", generator=g) >= args.null_p
    bits = torch.zeros((n + 63) // 64 * 8 + 8, dtype=torch.uint8, device="cuda")
    packed = (valid[: n // 8 * 8].view(-1, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(1)
    bits[: n // 8] = packed.to(torch.uint8)
    if n % 8:
        tail = sum(int(valid[n // 8 * 8 + k]) << k for k in range(n % 8))
        bits[n // 8] = tail
    nulls = int(n - valid.sum())
    ns = us * 1000
    torch.cuda.synchronize()
    ctx.sync()
    t_us, t_ns = pa.timestamp("us"), pa.timestamp("ns")
    d_us = DeviceArray.from_pointers(ctx, t_us, n, us.data_ptr(), validity_ptr=bits.data_ptr(), null_count=nulls,
                                     keepalive=(us, bits))
    d_ns = DeviceArray.from_pointers(ctx, t_ns, n, ns.data_ptr(), validity_ptr=bits.data_ptr(), null_count=nulls,
                                     keepalive=(ns, bits))
    cases = {
        "year": (lambda: bc.year(d_us), 8 + 8),
        "hour": (lambda: bc.hour(d_us), 8 + 8),
        "subsecond": (lambda: bc.subsecond(d_us), 8 + 8),
        "cast_ts_us_to_date32": (lambda: _cast(ctx, d_us, t_us, pa.date32()), 8 + 4),
        "cast_ts_ns_to_ts_us": (lambda: _cast(ctx, d_ns, t_ns, t_us), 8 + 8),
    }
    m = min(n, 1 << 20)
    host_us = pa.array(us[:m].cpu().numpy(), t_us, mask=~valid[:m].cpu().numpy())
    host_ns = pa.array(ns[:m].cpu().numpy(), t_ns, mask=~valid[:m].cpu().numpy())
    want = {
        "year": pc.year(host_us), "hour": pc.hour(host_us), "subsecond": pc.subsecond(host_us),
        "cast_ts_us_to_date32": pc.cast(host_us, pa.date32()), "cast_ts_ns_to_ts_us": pc.cast(host_ns, t_us),
    }
    info = _gpu_info()
    for name, (fn, data_bytes) in cases.items():
        out = fn()
        parity = out.slice(0, m).to_arrow().equals(want[name])
        del out
        fn()
        ctx.sync()
        # the calls run on the context's own stream: the events are recorded there
        stream = torch.cuda.ExternalStream(ctx.lib.b2_context_stream(ctx.handle))
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
        bpr = data_bytes + 0.25
        print(json.dumps({"case": name, "rows": n, "null_p": args.null_p, "median_ms": round(ms, 3),
                          "bytes_per_row": bpr, "GB_per_s": round(bpr * n / ms / 1e6, 1), "parity": parity,
                          "gpu": info}), flush=True)


if __name__ == "__main__":
    main()
