"""Throughput of the device argsort of Frame.sort (csrc/sort.cu) and of the row gather that follows it.

    python tools/bench_sort.py [--rows 1e8,1e9] [--string-rows 1e8] [--distinct 1e3,1e6] [--reps 3] [--cpu-rows 1e7] [--out result.json]

Workloads (keys device-resident unless said otherwise, seeded):
  f32          one float32 key, standard normal
  i64          one int64 key, uniform over [-2^62, 2^62)
  i32_f64      [int32 uniform over [0, 1e6) ascending, float64 standard normal descending]
  f32_nan_mask one float32 key with 1 % NaN and 1 % masked rows (a device mask)
  str_<d>      host arrow strings ("s" + a uniform number below d), --string-rows rows
Per workload, timed with CUDA events, best of --reps after a warm-up: `argsort` (b200_argsort: encode + radix passes), for strings
`rank` (the device string set, the host sort of the distinct strings and the rank column), and `take` (join.gather of two device
payload columns, float32 and int32, by the permutation).  A separate profiled run (torch.profiler) gives the kernel times: encode,
the number of radix passes and the time per pass (histogram + scan + scatter).  Algorithmic bytes: encode reads the keys and
writes 16 B/row (8 B more per row when a round reads through the permutation); a radix pass reads 8 + 16 B/row and writes 16 B/row;
their share of 3.35 TB/s (the H100 SXM data sheet) is printed beside each.  CPU baseline: pa.compute.sort_indices on the host over
the first --cpu-rows rows of the same keys, wall clock.  Every line names the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12
PASS_BYTES = 8 + 16 + 16


def best(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        del out
    return min(ms)


def kernel_times(fn):
    """{kernel: (launches, total ms)} of one call, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in ("k_sort_encode", "k_radix_hist", "k_scan_u32", "k_radix_scatter"):
            if k in e.name:
                c, t = out.get(k, (0, 0.0))
                out[k] = (c + 1, t + e.device_time_total / 1e3)
    return out


def workload(name, n, distinct, g):
    """(keys for sort.argsort, host copies of the keys for the CPU baseline, rank fn or None)"""
    import torch
    from vaex_b200 import _lib
    from vaex_b200 import sort as S
    dev = "cuda"
    if name == "f32":
        x = torch.randn(n, device=dev, generator=g)
        return [S.Key(x, _lib.F32)], [(x, None, False)], None
    if name == "i64":
        x = torch.randint(-2 ** 62, 2 ** 62, (n,), device=dev, generator=g, dtype=torch.int64)
        return [S.Key(x, _lib.I64)], [(x, None, False)], None
    if name == "i32_f64":
        a = torch.randint(0, 10 ** 6, (n,), device=dev, generator=g, dtype=torch.int32)
        b = torch.randn(n, device=dev, generator=g, dtype=torch.float64)
        return [S.Key(a, _lib.I32), S.Key(b, _lib.F64, descending=True)], [(a, None, False), (b, None, True)], None
    if name == "f32_nan_mask":
        x = torch.randn(n, device=dev, generator=g)
        x[torch.rand(n, device=dev, generator=g) < 0.01] = float("nan")
        m = (torch.rand(n, device=dev, generator=g) < 0.01).to(torch.uint8)
        return [S.Key(x, _lib.F32, mask=m)], [(x, m, False)], None
    import pyarrow as pa
    rng = np.random.default_rng(0)
    words = pa.array(["s%d" % i for i in range(distinct)], type=pa.large_string())
    col = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, distinct, n)), words).dictionary_decode()
    return None, [(col, None, False)], lambda: S.stage_key(col, n, False)


def cpu_baseline(host_keys, rows):
    import pyarrow as pa
    import pyarrow.compute as pc
    cols = {}
    for i, (x, m, _) in enumerate(host_keys):
        if isinstance(x, (pa.Array, pa.ChunkedArray)):
            cols[f"k{i}"] = x[:rows]
            continue
        v = x[:rows].cpu().numpy()
        cols[f"k{i}"] = pa.array(np.ma.array(v, mask=m[:rows].cpu().numpy().astype(bool)) if m is not None else v)
    table = pa.table(cols)
    keys = [(f"k{i}", "descending" if d else "ascending") for i, (_, _, d) in enumerate(host_keys)]
    t0 = time.perf_counter()
    pc.sort_indices(table, sort_keys=keys)
    s = time.perf_counter() - t0
    return dict(rows=rows, seconds=s, rows_per_s=rows / s, pyarrow=pa.__version__, pyarrow_cpu_count=pa.cpu_count(), host_cpus=os.cpu_count())


def run(name, n, distinct, reps, cpu_rows, card):
    import torch
    from vaex_b200 import join as J
    from vaex_b200 import sort as S
    g = torch.Generator(device="cuda").manual_seed(0)
    keys, host_keys, rank = workload(name, n, distinct, g)
    res = dict(workload=name if distinct is None else f"str_{distinct:g}", rows=n, device=card)
    if rank is not None:
        res["rank_ms"] = best(rank, reps)
        keys = [rank()]
    keysize = sum(k.data.element_size() if hasattr(k.data, "element_size") else k.data.dtype.itemsize for k in keys)
    res["argsort_ms"] = best(lambda: S.argsort(keys, n), reps)
    kt = kernel_times(lambda: S.argsort(keys, n))
    enc_n, enc_ms = kt.get("k_sort_encode", (0, 0.0))
    passes = kt.get("k_radix_scatter", (0, 0.0))[0]
    pass_ms = sum(kt.get(k, (0, 0.0))[1] for k in ("k_radix_hist", "k_scan_u32", "k_radix_scatter"))
    enc_bytes = n * (keysize + 16) + (enc_n - 1) * n * 8
    res.update(rounds=enc_n, encode_ms=enc_ms, encode_share=enc_bytes / (enc_ms * 1e-3) / PEAK if enc_ms else None, radix_passes=passes,
               ms_per_pass=pass_ms / passes if passes else 0.0, bytes_per_pass=PASS_BYTES * n,
               pass_share=PASS_BYTES * n / (pass_ms / passes * 1e-3) / PEAK if passes else None)
    perm = S.argsort(keys, n)
    payload = {"a": torch.randn(n, device="cuda", generator=g), "b": torch.randint(0, 1 << 30, (n,), device="cuda", generator=g, dtype=torch.int32)}
    res["take_ms"] = best(lambda: J.gather(payload, perm, n, lambda c: True), reps)
    res["take_share"] = n * (8 + 2 * 4 + 2 * 4) / (res["take_ms"] * 1e-3) / PEAK
    res["rows_per_s"] = n / ((res["argsort_ms"] + res.get("rank_ms", 0.0)) * 1e-3)
    if cpu_rows:
        res["cpu_sort_indices"] = cpu_baseline(host_keys, min(cpu_rows, n))
    del keys, host_keys, perm, payload
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1e8,1e9")
    ap.add_argument("--workloads", default="f32,i64,i32_f64,f32_nan_mask")
    ap.add_argument("--string-rows", default="1e8")
    ap.add_argument("--distinct", default="1e3,1e6")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-rows", type=float, default=1e7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sort needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    plan = [(w, int(float(n)), None) for n in a.rows.split(",") if n for w in a.workloads.split(",") if w]
    plan += [("str", int(float(n)), int(float(d))) for n in a.string_rows.split(",") if n for d in a.distinct.split(",") if d]
    results = []
    for w, n, d in plan:
        try:
            r = run(w, n, d, a.reps, int(a.cpu_rows), card)
        except (torch.cuda.OutOfMemoryError, MemoryError, RuntimeError) as e:
            torch.cuda.empty_cache()
            r = dict(workload=w, rows=n, distinct=d, device=card, skipped=str(e).splitlines()[0][:200])
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
