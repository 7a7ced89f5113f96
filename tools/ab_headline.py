#!/usr/bin/env python
"""A/B timing of the headline kernel pair on ONE box: count(*) binby=[x,y], shape 1024, fp32, device-resident rows.

    VAEX_B200_LIB=/path/to/other/libb200agg.so python tools/ab_headline.py [--rows 1e9] [--reps 10]

Box-to-box variation between gpurun calls is ~5 % (the same unchanged kernel differs that much), so kernel variants are only
compared inside one call: run this script once per library build.  Prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--tag", default="")
    ap.add_argument("--occupy", default="", help="CTAS,MICROSECONDS: a do-nothing kernel holding that many SMs (1024 threads, 200 KB of shared memory "
                                                "each) is released on another slot's stream at the moment the timed pass starts — what an NCCL all-reduce of "
                                                "the previous step does to the partition kernel on a multi-GPU run")
    args = ap.parse_args()
    import torch
    from vaex_b200 import _lib, engine, superagg
    n = int(args.rows)
    ctx = _lib.context(0)
    g = torch.Generator(device="cuda").manual_seed(42)
    x = torch.randn(n, device="cuda", dtype=torch.float32, generator=g)
    y = torch.randn(n, device="cuda", dtype=torch.float32, generator=g)
    bx = superagg.BinnerScalar_float32(1, "x", -3, 3, 1024)
    by = superagg.BinnerScalar_float32(1, "y", -3, 3, 1024)
    grid = superagg.Grid([bx, by])
    agg = superagg.AggCount_float32(grid, 1, 1)
    bx.set_data(0, x)
    by.set_data(0, y)
    stream = engine.slot_stream(ctx, 0)
    times = []
    for rep in range(args.reps + 3):
        agg.reset(0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            if args.occupy:
                ctas, usec = (int(v) for v in args.occupy.split(","))
                engine.slot_stream(ctx, 1).wait_event(e0)
                _lib.check(_lib.lib().b200_ctx_occupy(ctx._h, 1, ctas, 1024, 200 * 1024, usec * 1000))
            grid.bin(0, [agg], n)
            e1.record()
        ctx.sync()
        if rep >= 3:
            times.append(e0.elapsed_time(e1))
    res = agg.get_result()
    total = int(res.sum())
    import hashlib
    sha = hashlib.sha1(res.tobytes()).hexdigest()[:16]
    times.sort()
    print(json.dumps({"tag": args.tag, "lib": os.path.basename(_lib.LIB_PATH), "path": "ring", "rows": n, "occupy": args.occupy or None,
                      "ms_min": times[0], "ms_median": times[len(times) // 2], "rows_per_s_median": n / (times[len(times) // 2] * 1e-3), "count_ok": total == n, "grid_sha": sha}))


if __name__ == "__main__":
    main()
