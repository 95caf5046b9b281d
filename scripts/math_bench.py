"""Time the numeric math kernels on the device with CUDA events, and a Filter in the same run as an anchor: abs / sqrt (of |x|) /
round(x, 2) over float64, round(x, 2, half_to_even) over float32, round_to_multiple(x, 1000) / power(x, 3) / abs over
int64, bit_wise_and against a scalar and shift_right.  Each line gives the median time, the algorithmic bytes per row
(a unary float64 map with a nullable input and output reads 8.125 B/row and writes 8.125 B/row; the scalar operand of a
binary op is not counted), that rate as a share of the H100 SXM data sheet's 3.35 TB/s, a parity flag (the device
against pyarrow.compute on a 1M-row prefix), and the card's name and power limit read in the same run.

    python scripts/math_bench.py --rows 1000000000 --null-p 0.1 --iters 10
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
    g = torch.Generator(device="cuda").manual_seed(3)
    valid, bits, nulls = _validity(n, args.null_p, g)
    f64 = (torch.rand(n, device="cuda", dtype=torch.float64, generator=g) - 0.5) * 2e6
    f32 = f64.to(torch.float32)
    i64 = torch.randint(-(1 << 40), 1 << 40, (n,), device="cuda", dtype=torch.int64, generator=g)
    small = torch.randint(-1000, 1000, (n,), device="cuda", dtype=torch.int64, generator=g)
    mask = torch.rand(n, device="cuda", generator=g) < 0.5
    mask_bits = torch.zeros((n + 63) // 64 * 8 + 8, dtype=torch.uint8, device="cuda")
    full = n // 8 * 8
    mask_bits[: n // 8] = (mask[:full].view(-1, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(1).to(torch.uint8)
    torch.cuda.synchronize()

    def dev(t, ty):
        return DeviceArray.from_pointers(ctx, ty, n, t.data_ptr(), validity_ptr=bits.data_ptr(), null_count=nulls, keepalive=(t, bits))

    nonneg = f64.abs()
    d64, d32, di, ds = dev(f64, pa.float64()), dev(f32, pa.float32()), dev(i64, pa.int64()), dev(small, pa.int64())
    dpos = dev(nonneg, pa.float64())
    dmask = DeviceArray.from_pointers(ctx, pa.bool_(), n, mask_bits.data_ptr(), keepalive=(mask_bits,))
    three = pa.scalar(3, pa.int64())
    # name: (call, pyarrow call on the prefix, bytes per row in + out, validity included)
    cases = {
        "filter float64 (anchor)": (lambda: bc.filter(d64, dmask), None, None),
        "abs float64": (lambda: bc.abs(d64), lambda x: pc.abs(x["f64"]), 16.25),
        "sqrt float64": (lambda: bc.sqrt(dpos), lambda x: pc.sqrt(x["pos"]), 16.25),
        "round(x, 2) float64": (lambda: bc.round(d64, 2), lambda x: pc.round(x["f64"], 2), 16.25),
        "round(x, 2, half_to_even) float32": (lambda: bc.round(d32, 2, "half_to_even"), lambda x: pc.round(x["f32"], 2), 8.25),
        "abs int64": (lambda: bc.abs(di), lambda x: pc.abs(x["i64"]), 16.25),
        "round_to_multiple(x, 1000) int64": (lambda: bc.round_to_multiple(di, 1000),
                                             lambda x: pc.round_to_multiple(x["i64"], pa.scalar(1000, pa.int64())), 16.25),
        "power(x, 3) int64": (lambda: bc.power(ds, three), lambda x: pc.power(x["small"], three), 16.25),
        "bit_wise_and(x, 0xffff) int64": (lambda: bc.bit_wise_and(di, pa.scalar(0xFFFF, pa.int64())),
                                          lambda x: pc.bit_wise_and(x["i64"], pa.scalar(0xFFFF, pa.int64())), 16.25),
        "shift_right(x, 4) int64": (lambda: bc.shift_right(di, pa.scalar(4, pa.int64())),
                                    lambda x: pc.shift_right(x["i64"], pa.scalar(4, pa.int64())), 16.25),
    }
    m = min(n, 1 << 20)
    hmask = ~valid[:m].cpu().numpy()
    host = {"f64": pa.array(f64[:m].cpu().numpy(), mask=hmask), "pos": pa.array(nonneg[:m].cpu().numpy(), mask=hmask), "f32": pa.array(f32[:m].cpu().numpy(), mask=hmask),
            "i64": pa.array(i64[:m].cpu().numpy(), mask=hmask), "small": pa.array(small[:m].cpu().numpy(), mask=hmask)}
    stream = torch.cuda.ExternalStream(ctx.lib.b2_context_stream(ctx.handle))
    for name, (fn, ref, bpr) in cases.items():
        out = fn()
        parity = None if ref is None else out.slice(0, m).to_arrow().equals(ref(host))
        if bpr is None:  # the filter: values and validity in, the mask in, the selected values and validity out
            sel = out.length
            bpr = 8 + 0.125 + 0.125 + (8 + 0.125) * sel / n
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
