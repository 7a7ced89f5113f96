"""Throughput of the string calls of device expressions (csrc/strexpr.cu) and of a string filter end to end.

    python tools/bench_str_expr.py [--rows 1e8] [--means 8,32,64,128,256] [--e2e-means 8,32,256] [--reps 5] [--e2e-rows 1e8]
                                   [--e2e-max-gb 6] [--groupby-rows 1e8] [--out result.json]

Kernel: for each mean row length, --rows rows of random lowercase bytes (lengths uniform in [0, 2 * mean]) built on the device as an
arrow large_string layout; each function is one b200_str_eval call over the device buffers, timed with CUDA events on the slot's
stream around --reps calls after a warm-up.  count is timed in both of its forms, one thread per row and one warp per row
(B200_STR_SCAN), and in the form the call picks.  Algorithmic bytes: the offsets (8 B/row) plus, for the calls that read every byte,
the bytes; their share of 3.35 TB/s (the H100 SXM data sheet) is printed.
End to end, from host memory, wall clock: Frame({"s": host arrow}, filter="str_contains(s, 'abc', regex=False)").count() per
--e2e-means, with the rows capped so that the strings stay under --e2e-max-gb; and a string filter with a string groupby key on one
frame, Frame({"city": host arrow}, filter="str_contains(city, 'burg', regex=False)").groupby("city", agg="count") over --groupby-rows
rows of 16 city names, beside the same groupby without the filter.  Every line names the card and its power limit."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12
CALLS = [("equals", b"abcdefgh", False), ("startswith", b"abc", False), ("endswith", b"xyz", False), ("len", b"", True),
         ("byte_length", b"", False), ("contains", b"abc", True), ("count", b"ab", True), ("find", b"abc", True), ("rfind", b"abc", True)]
SCANS = ("count",)  # the one call with two kernel forms


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def device_strings(n, mean, seed=0):
    """n rows of bytes a..z with lengths uniform in [0, 2 * mean], as int64 offsets + bytes on the device"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    lens = torch.randint(0, 2 * mean + 1, (n,), device="cuda", generator=g, dtype=torch.int64)
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=off[1:])
    nbytes = int(off[-1])
    data = torch.randint(ord("a"), ord("z") + 1, (nbytes + 16,), device="cuda", generator=g, dtype=torch.uint8)
    return off, data, nbytes


def time_call(ctx, op, off, data, nbytes, pattern, plen, n, out, reps):
    """ms per call: CUDA events on slot 0's stream, where b200_str_eval runs"""
    import torch
    from vaex_b200 import _lib
    L = _lib.lib()
    end = (1 << 63) - 1
    st = torch.cuda.ExternalStream(ctx.stream(0))

    def run():
        _lib.check(L.b200_str_eval(ctx._h, 0, op, off.data_ptr(), 8, data.data_ptr(), None, None, 0, None, None, pattern, plen, 0, end, n, nbytes,
                                   out.data_ptr()))
    run()
    ctx.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(reps):
        run()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def kernels(args, gpu):
    import torch
    from vaex_b200 import _lib, expression as X
    ctx = _lib.context()
    n = int(float(args.rows))
    results = []
    for mean in [int(m) for m in args.means.split(",")]:
        off, data, nbytes = device_strings(n, mean)
        out = torch.empty(n * 8, dtype=torch.uint8, device="cuda")
        for name, pattern, reads_all in CALLS:
            op = getattr(X, "EX_STR_" + name.upper())
            dpat = torch.frombuffer(bytearray(pattern or b"\0"), dtype=torch.uint8).cuda()
            forms = [None, "thread", "warp"] if name in SCANS else [None]
            for form in forms:
                if form:
                    os.environ["B200_STR_SCAN"] = form
                else:
                    os.environ.pop("B200_STR_SCAN", None)
                s = time_call(ctx, op, off, data, nbytes, C.c_void_p(dpat.data_ptr()), len(pattern), n, out, args.reps)
                moved = 8 * (n + 1) + (nbytes if reads_all else 0)
                r = dict(kind="kernel", mean=mean, rows=n, call=name, form=form or "picked", ms=s * 1e3, rows_per_s=n / s, bytes=moved,
                         share_of_hbm=moved / s / PEAK, gpu=gpu)
                results.append(r)
                print(json.dumps(r), flush=True)
        os.environ.pop("B200_STR_SCAN", None)
        del off, data, out
        torch.cuda.empty_cache()
    return results


def end_to_end(args, gpu):
    import pyarrow as pa
    from vaex_b200.frame import Frame
    results = []
    rng = np.random.default_rng(1)
    for mean in [int(m) for m in args.e2e_means.split(",")]:
        n = int(min(float(args.e2e_rows), args.e2e_max_gb * 1e9 / max(mean, 1)))
        lens = rng.integers(0, 2 * mean + 1, n)
        off = np.zeros(n + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        data = rng.integers(ord("a"), ord("z") + 1, int(off[-1]), dtype=np.uint8)
        arr = pa.Array.from_buffers(pa.large_string(), n, [None, pa.py_buffer(off), pa.py_buffer(data)])
        df = Frame({"s": arr}, filter="str_contains(s, 'abc', regex=False)")
        df.count()  # warm-up: module load, buffers
        ts = []
        for _ in range(max(1, args.reps // 2)):
            t = time.perf_counter()
            got = df.count()
            ts.append(time.perf_counter() - t)
        s = min(ts)
        moved = off.nbytes + data.nbytes
        r = dict(kind="end_to_end", mean=mean, rows=n, ms=s * 1e3, rows_per_s=n / s, host_bytes=moved, gb_per_s=moved / s / 1e9, kept=int(got),
                 gpu=gpu)
        results.append(r)
        print(json.dumps(r), flush=True)
        del arr, df, data, off
    return results


def groupby_filtered(args, gpu):
    import pyarrow as pa
    from vaex_b200.frame import Frame
    n = int(float(args.groupby_rows))
    names = ["Hamburg", "Augsburg", "Duisburg", "Amsterdam", "Rotterdam", "Utrecht", "Berlin", "Munich", "Cologne", "Frankfurt",
             "Strasbourg", "Luxembourg", "Edinburgh", "Paris", "Lyon", "Nice"]
    codes = np.random.default_rng(2).integers(0, len(names), n).astype(np.int32)
    city = pa.DictionaryArray.from_arrays(pa.array(codes), pa.array(names, pa.large_string())).cast(pa.large_string())
    results = []
    for filt in ("str_contains(city, 'burg', regex=False)", None):
        df = Frame({"city": city}, filter=filt)
        df.groupby("city", agg="count")  # warm-up
        ts = []
        for _ in range(2):
            t = time.perf_counter()
            out = df.groupby("city", agg="count")
            ts.append(time.perf_counter() - t)
        s = min(ts)
        r = dict(kind="groupby", filter=filt, rows=n, ms=s * 1e3, rows_per_s=n / s, groups=len(out["count"]), kept=int(np.sum(out["count"])),
                 host_bytes=city.nbytes, gpu=gpu)
        results.append(r)
        print(json.dumps(r), flush=True)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1e8")
    ap.add_argument("--means", default="8,32,64,128,256")
    ap.add_argument("--e2e-means", default="8,32,256")
    ap.add_argument("--groupby-rows", default="1e8")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--e2e-rows", default="1e8")
    ap.add_argument("--e2e-max-gb", type=float, default=6.0)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_str_expr.py needs a GPU")
    gpu = card()
    results = kernels(args, gpu) + end_to_end(args, gpu) + groupby_filtered(args, gpu)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
