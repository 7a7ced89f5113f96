"""Throughput of Frame.groupby over calendar periods (BinnerTime: the period computed in k_binby from the raw ticks).

    python tools/bench_groupby_binners.py [--rows 1e9] [--reps 3] [--host-rows 1e8] [--check-rows 1e7] [--out result.json]

Workload (seeded, device-resident): `t` int64-ns datetimes uniform over 2000-01-01 .. 2024-01-01, `y` float32 standard normal.
  per_month / per_day   groupby(BinnerTime.per_month('t') / per_day('t'), agg={'y': 'sum'}), the binner built once (its limits pass
                        is timed apart as `limits`)
  hash_<card>           groupby('k', agg={'y': 'sum'}) on an int64 key uniform over as many values as the period grid has cells
                        (288 months, 8766 days): the hashed-key path the time binner replaces
  numpy_<res>           the period codes computed by numpy on the host, (t.astype('M8[R]') - begin).astype(int), over --host-rows
                        rows: what a user without the time binner would compute and then group
Device times: best of --reps after a warm-up, host clock around a synchronised call.  Before timing, the first --check-rows rows are
grouped on the device and compared with numpy.  Every line names the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LO, HI = np.datetime64("2000-01-01", "ns").astype(np.int64), np.datetime64("2024-01-01", "ns").astype(np.int64)


class DeviceDatetime:
    """a datetime64[ns] column in device memory: a torch int64 tensor exposed with the datetime typestr"""

    def __init__(self, tensor):
        self.t, self.dtype = tensor, np.dtype("M8[ns]")
        self.__cuda_array_interface__ = dict(tensor.__cuda_array_interface__, typestr=self.dtype.str)

    def __len__(self):
        return len(self.t)

    def __getitem__(self, s):
        return DeviceDatetime(self.t[s])


def best(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return min(times)


def check(t, y, n):
    """the first n rows grouped per month and per day on the device against numpy"""
    from vaex_b200.frame import BinnerTime, Frame
    df = Frame({"t": DeviceDatetime(t[:n]), "y": y[:n]})
    tt, yy = t[:n].cpu().numpy().view("M8[ns]"), y[:n].cpu().numpy().astype(np.float64)
    for res in ("M", "D"):
        out = df.groupby(BinnerTime("t", res, df=df), agg={"y": "sum"})
        f = tt.view(np.int64).astype(np.float32).astype(np.float64)
        begin, end = np.array([f.min(), f.max()]).astype("M8[ns]").astype(f"M8[{res}]")
        codes = (tt.astype(f"M8[{res}]") - begin).astype(np.int64)
        ok = (codes >= 0) & (codes <= (end - begin).astype(np.int64))
        want = np.bincount(codes[ok], weights=yy[ok])
        used = np.nonzero(np.bincount(codes[ok]))[0]
        assert np.array_equal(out["t"], begin + used), res
        assert np.allclose(out["y_sum"], want[used], rtol=1e-9, atol=1e-6), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-rows", type=float, default=1e8)
    ap.add_argument("--check-rows", type=float, default=1e7)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from vaex_b200.frame import BinnerTime, Frame
    n = int(a.rows)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    g = torch.Generator(device="cuda").manual_seed(0)
    t = torch.randint(int(LO), int(HI), (n,), device="cuda", generator=g, dtype=torch.int64)
    y = torch.randn(n, device="cuda", generator=g, dtype=torch.float32)
    check(t, y, min(n, int(a.check_rows)))
    df = Frame({"t": DeviceDatetime(t), "y": y})
    results = []

    def report(name, seconds, rows):
        r = {"workload": name, "rows": rows, "seconds": round(seconds, 4), "rows_per_s": rows / seconds, "card": card}
        results.append(r)
        print(json.dumps(r), flush=True)

    t0 = time.perf_counter()
    BinnerTime.per_month("t", df=df)
    torch.cuda.synchronize()
    report("limits", time.perf_counter() - t0, n)
    host_n = min(n, int(a.host_rows))
    th = t[:host_n].cpu().numpy().view("M8[ns]")
    for name, res in (("per_month", "M"), ("per_day", "D")):
        b = BinnerTime("t", res, df=df)
        report(name, best(lambda: df.groupby(b, agg={"y": "sum"}), a.reps), n)
        k = torch.randint(0, b.N, (n,), device="cuda", generator=g, dtype=torch.int64)
        dk = Frame({"k": k, "y": y})
        report(f"hash_{b.N}", best(lambda: dk.groupby("k", agg={"y": "sum"}), a.reps), n)
        del k, dk
        begin = np.datetime64(b.begin, res)
        t0 = time.perf_counter()
        (th.astype(f"M8[{res}]") - begin).astype(np.int64)
        report(f"numpy_{res}", time.perf_counter() - t0, host_n)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
