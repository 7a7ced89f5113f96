"""Throughput of the device index_hash: index build, map_index and the duplicate expansion (map_index_duplicates); and of the
end-to-end Frame.join (index build, lookup pass, gather of the right's payload, the whole join).

    python tools/bench_join.py [--left 1e8,1e9] [--right 1e3,1e6,1e8] [--dup 0,0.1,1] [--reps 3] [--out result.json]
                               [--join-left 1e9] [--join-right 1e6,1e8] [--skip-index]

Frame.join phase: a device-resident int64 left key against a right side of unique int64 keys with two numeric payload columns
(float64, int32) and one string payload column (1000 distinct short strings, host arrow).  Every left key matches, so the numeric
columns stay on the device and the string column comes back as a host arrow array.  Wall clock around each phase, which ends in a
device synchronise; median of `--reps` after a warm-up.

Right keys: right_n / (1 + dup) distinct int64 keys, the rest repeats of them (dup = 0.1: every tenth row repeats a key; dup = 1:
every key twice on average), shuffled, device-resident.  Left keys: uniform over 1.1x the distinct keys (about 9 % find nothing).
Every phase is warmed up at its shape, then timed `--reps` times with CUDA events; min / median / max are reported.  The CPU
baseline is the compiled reference's index_hash_int64 (oracle/_ref) at one thread on a 1e6-row right side and 1e7 left rows.
Prints one JSON line per configuration, then the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps):
    import torch
    fn()  # warm-up at this shape
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
    ms.sort()
    return dict(min_ms=ms[0], median_ms=ms[len(ms) // 2], max_ms=ms[-1])


def keys(left_n, right_n, dup, seed=0):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    distinct = max(1, int(round(right_n / (1 + dup))))
    base = torch.randperm(distinct, device="cuda", generator=g).to(torch.int64)
    extra = torch.randint(0, distinct, (right_n - distinct,), device="cuda", generator=g)
    right = torch.cat([base, extra])[torch.randperm(right_n, device="cuda", generator=g)] * 7919 + 3
    left = torch.randint(0, int(distinct * 1.1) + 1, (left_n,), device="cuda", generator=g) * 7919 + 3
    return left, right


def run_config(left_n, right_n, dup, reps):
    import torch
    from vaex_b200 import superutils
    left, right = keys(left_n, right_n, dup)

    def build():
        h = superutils.index_hash_int64(1)
        h.update(right, 0)
        return h

    res = dict(left_rows=left_n, right_rows=right_n, dup=dup)
    res["build"] = timed(build, reps)
    h = build()
    res["has_duplicates"] = h.has_duplicates
    out = torch.empty(left_n, dtype=torch.int64, device="cuda")
    res["map_index"] = timed(lambda: h.map_index(left, out), reps)
    h.map_index_duplicates(left[:1], 0)  # the first call after a change sorts the row log (timed on its own below)
    if h.has_duplicates:  # once per change: no warm-up possible, one fresh index per sample
        ms = []
        for _ in range(reps):
            h2 = build()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            h2.map_index_duplicates(left[:1], 0, device=True)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
            del h2
        ms.sort()
        res["overflow_sort"] = dict(min_ms=ms[0], median_ms=ms[len(ms) // 2], max_ms=ms[-1])
    pairs = h.map_index_duplicates(left, 0, device=True)
    res["pairs"] = int(pairs[0].shape[0])
    del pairs
    res["duplicates"] = timed(lambda: h.map_index_duplicates(left, 0, device=True), reps)
    for k, n in (("build", right_n), ("map_index", left_n), ("duplicates", left_n)):
        res[k]["rows_per_s"] = n / (res[k]["median_ms"] * 1e-3)
    del h, out, left, right
    torch.cuda.empty_cache()
    return res


def run_frame_join(left_n, right_n, reps):
    import pyarrow as pa
    import torch
    from vaex_b200 import join as J
    from vaex_b200 import execution, taskpart
    from vaex_b200.frame import Frame
    g = torch.Generator(device="cuda").manual_seed(1)
    rk = torch.randperm(right_n, device="cuda", generator=g).to(torch.int64) * 7919 + 3
    lk = torch.randint(0, right_n, (left_n,), device="cuda", generator=g) * 7919 + 3
    words = np.array(["w%d" % i for i in range(1000)], dtype=object)
    right = {"k": rk, "a": torch.rand(right_n, device="cuda", dtype=torch.float64, generator=g),
             "b": torch.randint(0, 1 << 30, (right_n,), device="cuda", generator=g).to(torch.int32),
             "s": pa.array(words[np.arange(right_n) % 1000].tolist(), type=pa.large_string())}
    left, rframe = Frame({"k": lk}), Frame(right)

    def wall(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
            del out
        ms.sort()
        return dict(min_ms=ms[0], median_ms=ms[len(ms) // 2], max_ms=ms[-1])

    res = dict(left_rows=left_n, right_rows=right_n, payload="float64, int32 (device), large_string (host arrow)")
    res["build"] = wall(lambda: rframe._index("k"))
    ix = rframe._index("k")
    lookup = torch.empty(left_n, dtype=torch.int32 if right_n < 2 ** 31 else torch.int64, device="cuda")

    def lookup_pass():
        part = taskpart.TaskPartLookup(ix, "k", lookup, False)
        execution.Executor().execute({"k": lk}, [execution.Task(part)], left_n)
    res["lookup"] = wall(lookup_pass)
    res["gather_numeric"] = wall(lambda: J.gather({"a": right["a"], "b": right["b"]}, lookup, right_n, lambda c: True))
    res["gather_string"] = wall(lambda: J.gather({"s": right["s"]}, lookup, right_n, lambda c: True))
    res["join"] = wall(lambda: left.join(rframe, on="k"))
    res["join"]["rows_per_s"] = left_n / (res["join"]["median_ms"] * 1e-3)
    del ix, lookup, left, rframe, right, lk, rk
    torch.cuda.empty_cache()
    return res


def cpu_baseline():
    from oracle import ref_driver
    if not ref_driver.available():
        return dict(skipped="oracle/_ref not built")
    su = ref_driver.modules()[1]
    rng = np.random.default_rng(0)
    right = rng.integers(0, 500_000, 10 ** 6) * 7919 + 3
    left = rng.integers(0, 550_000, 10 ** 7) * 7919 + 3
    h = su.index_hash_int64(1)
    t0 = time.perf_counter()
    h.update(right, 0)
    t1 = time.perf_counter()
    h.map_index(left)
    t2 = time.perf_counter()
    h.map_index_duplicates(left, 0)
    t3 = time.perf_counter()
    return dict(threads=1, right_rows=len(right), left_rows=len(left), dup=1.0, build_rows_per_s=len(right) / (t1 - t0),
                map_index_rows_per_s=len(left) / (t2 - t1), duplicates_rows_per_s=len(left) / (t3 - t2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--left", default="1e8,1e9")
    ap.add_argument("--right", default="1e3,1e6,1e8")
    ap.add_argument("--dup", default="0,0.1,1")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--join-left", default="1e9")
    ap.add_argument("--join-right", default="1e6,1e8")
    ap.add_argument("--skip-index", action="store_true", help="only the Frame.join phase")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_join needs a GPU")
    results = []
    for ln in ([] if a.skip_index else (int(float(x)) for x in a.left.split(","))):
        for rn in (int(float(x)) for x in a.right.split(",")):
            for d in (float(x) for x in a.dup.split(",")):
                try:
                    r = run_config(ln, rn, d, a.reps)
                except (torch.cuda.OutOfMemoryError, MemoryError, RuntimeError) as e:
                    torch.cuda.empty_cache()
                    r = dict(left_rows=ln, right_rows=rn, dup=d, skipped=str(e).splitlines()[0][:200])
                print(json.dumps(r), flush=True)
                results.append(r)
    for ln in (int(float(x)) for x in a.join_left.split(",")):
        for rn in (int(float(x)) for x in a.join_right.split(",")):
            try:
                r = dict(frame_join=run_frame_join(ln, rn, a.reps))
            except (torch.cuda.OutOfMemoryError, MemoryError, RuntimeError) as e:
                torch.cuda.empty_cache()
                r = dict(frame_join=dict(left_rows=ln, right_rows=rn, skipped=str(e).splitlines()[0][:200]))
            print(json.dumps(r), flush=True)
            results.append(r)
    base = cpu_baseline() if not a.skip_index else dict(skipped="--skip-index")
    print(json.dumps(dict(cpu_baseline=base)), flush=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=card)), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(results=results, cpu_baseline=base, device=card), f, indent=1)


if __name__ == "__main__":
    main()
