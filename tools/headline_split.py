#!/usr/bin/env python
"""Per-kernel split of the headline count: count(*) binby=[x,y], shape 1024, fp32, device-resident N(0,1) rows.

    [VAEX_B200_LIB=/path/to/other/libb200agg.so] python tools/headline_split.py [--rows 1e9] [--reps 10]

Sets B200_RING_EVENTS=1, so csrc/ringcount.cu records CUDA events around the memset before a batch, k_ring_partition (K1) and
k_ring_count (K2) of every pass; b200_ctx_ring_times reads them back.  Prints one JSON line: the median milliseconds of each part
and each kernel's DRAM rate, K1 at 8 B/row of keys + 2 B per scratch entry written, K2 at 2 B per entry read (entries from
b200_ctx_path_stats, pads included).  Like tools/ab_headline.py, compare builds back to back on one GPU: machine-to-machine variation is ~5 %."""
import argparse
import hashlib
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
    args = ap.parse_args()
    os.environ["B200_RING_EVENTS"] = "1"
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
    parts = {"memset_ms": [], "k1_ms": [], "k2_ms": [], "pass_ms": []}
    for rep in range(args.reps + 3):
        agg.reset(0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            grid.bin(0, [agg], n)
            e1.record()
        ctx.sync()
        t = ctx.ring_times(0)
        if rep >= 3:
            for k in ("memset_ms", "k1_ms", "k2_ms"):
                parts[k].append(t[k])
            parts["pass_ms"].append(e0.elapsed_time(e1))
    st = ctx.path_stats(0)
    res = agg.get_result()
    med = {k: sorted(v)[len(v) // 2] for k, v in parts.items()}
    rows_b, entries = st["rows"], st["entries"]  # one batch up to 2^30 rows
    k1_bytes = rows_b * 8 + entries * 2
    k2_bytes = entries * 2
    out = {"tag": args.tag, "lib": os.path.basename(_lib.LIB_PATH), "rows": n, **med,
           "k1_gbs": k1_bytes / (med["k1_ms"] * 1e-3) / 1e9 if med["k1_ms"] else None,
           "k2_gbs": k2_bytes / (med["k2_ms"] * 1e-3) / 1e9 if med["k2_ms"] else None,
           "k1_bytes_per_row": k1_bytes / rows_b if rows_b else None, "k2_bytes_per_row": k2_bytes / rows_b if rows_b else None,
           "memset_bytes": st["memset_bytes"], "k1_ms_min": min(parts["k1_ms"]), "k2_ms_min": min(parts["k2_ms"]),
           "count_ok": int(res.sum()) == n, "grid_sha": hashlib.sha1(res.tobytes()).hexdigest()[:16]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
