"""Time the lasso selection on the H100 with CUDA events: b200_lasso over 1e8 float32 (cast by b200_eval) and float64 device rows for
4, 64, 1024 and 16384 vertices in both the plain and the banded loop, and count(binby=[x, y], shape=1024) with a lasso selection
against the same count without one.  Prints the card's name and power limit, then one line per case with its rows/s."""
import argparse
import subprocess
import sys
import os

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def timed(fn, reps, warmup=2, stream=None):
    """seconds per call: CUDA events on `stream` (the slot's stream the kernel is enqueued on), or around calls that return only
    when their results are read"""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(reps):
        fn()
    end.record(stream)
    end.synchronize()
    return start.elapsed_time(end) / 1e3 / reps


def main():
    import torch
    import lasso_oracle as L
    from vaex_b200 import _lib
    from vaex_b200.frame import Frame
    from vaex_b200.selections import LassoPlan, _Lasso
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("card:", card())
    n = a.rows
    g = torch.Generator(device="cuda").manual_seed(0)
    x64 = torch.rand(n, device="cuda", dtype=torch.float64, generator=g) * 3.2 - 1.6
    y64 = torch.rand(n, device="cuda", dtype=torch.float64, generator=g) * 3.2 - 1.6
    x32, y32 = x64.float(), y64.float()
    ctx = _lib.context()
    slot_stream = torch.cuda.ExternalStream(ctx.stream(ctx.slot(0)), device=f"cuda:{ctx.device}")
    for dtype, (x, y) in (("float64", (x64, y64)), ("float32", (x32, y32))):
        for nv in (4, 64, 1024, 16384):
            xs, ys = L.polygon(nv, seed=nv)
            for banded in (False, True):
                if dtype == "float32":
                    df = Frame({"x": x, "y": y})
                    df.select_lasso("x", "y", xs, ys)
                    lasso = df._selection(True).lassos[0][1]
                    lasso.plan = LassoPlan(xs, ys, banded=banded)
                else:
                    lasso = _Lasso(LassoPlan(xs, ys, banded=banded), x, y)
                if not banded and nv == 16384:
                    reps, rows = 1, n // 10
                else:
                    reps, rows = a.reps, n
                t = timed(lambda: lasso.chunk(0, 0, rows), reps, warmup=1, stream=slot_stream)
                ctx.sync()
                print(f"b200_lasso {dtype:7s} {nv:6d} vertices {'banded' if banded else 'plain ':6s}: {rows / t / 1e9:7.2f} G rows/s ({t * 1e3:.2f} ms"
                      f" for {rows} rows)", flush=True)
    df = Frame({"x": x32, "y": y32})
    xs, ys = L.polygon(64, seed=1)
    df.select_lasso("x", "y", xs, ys)
    kw = dict(binby=["x", "y"], limits=[[-1.6, 1.6]] * 2, shape=1024)
    t0 = timed(lambda: df.count(**kw), a.reps, warmup=1)
    t1 = timed(lambda: df.count(selection=True, **kw), a.reps, warmup=1)
    print(f"count(binby=[x, y], shape=1024) float32: {n / t0 / 1e9:.2f} G rows/s without a selection, {n / t1 / 1e9:.2f} G rows/s with a "
          f"64-vertex lasso (selection=True)")


if __name__ == "__main__":
    main()
