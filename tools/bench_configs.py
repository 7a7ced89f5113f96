#!/usr/bin/env python
"""Times every BASELINE.json configuration on one H100 with device-resident columns (the roofline setting) and prints one
JSON object per config: rows/s, achieved algorithmic GB/s (SURVEY.md 8d bytes/row) and the fraction of the measured HBM peak.

    python tools/bench_configs.py [--rows 1e9] [--configs C1,C2,C3,C4,C5,CV]

This is a companion to bench.py (which owns the headline line the driver parses); results are quoted in DESIGN.md.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--configs", default="C1,C5,C2,C3,C4")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from vaex_b200 import _lib, engine, superagg, superutils
    from vaex_b200.frame import Frame

    from bench import measured_peak
    peak, _ = measured_peak()
    ctx = _lib.context(0)
    stream = engine.slot_stream(ctx, 0)
    gen = torch.Generator(device="cuda").manual_seed(42)

    def timed(fn, reps, setup=None):
        """best of `reps` device times of fn(); setup() (e.g. a grid reset) runs and finishes before each timed window"""
        if setup:
            setup()
        fn()
        ctx.sync()
        torch.cuda.synchronize()
        best = None
        for _ in range(reps):
            if setup:
                setup()
                ctx.sync()
                torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            ctx.sync()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            best = ms if best is None else min(best, ms)
        return best

    def report(name, workload, rows, bytes_per_row, ms, **extra):
        gbs = rows * bytes_per_row / (ms * 1e-3) / 1e9
        print(json.dumps(dict(config=name, workload=workload, rows=rows, ms=ms, rows_per_s=rows / (ms * 1e-3), algorithmic_bytes_per_row=bytes_per_row,
                              achieved_gbs=gbs, frac_of_measured_hbm=gbs / peak, **extra)), flush=True)

    n = int(args.rows)
    for cfg in args.configs.split(","):
        torch.cuda.empty_cache()
        if cfg == "C1":
            rows = 10_000_000
            x = torch.empty(rows, dtype=torch.float64, device="cuda").normal_(generator=gen)
            b = superagg.BinnerScalar_float64(1, "x", -3.0, 3.0, 128)
            g = superagg.Grid([b])
            a = superagg.AggCount_int64(g, 1, 1)
            b.set_data(0, x)

            def run():
                a.reset(0)
                g.bin(0, [a], rows)
            ms = timed(run, args.reps)
            assert int(a.get_result().sum()) == rows
            report("C1", "df.count(binby=x, shape=128) on 1e7 fp64 rows (shared-memory privatised)", rows, 8, ms)
        elif cfg == "CV":
            # legacy statistics (csrc/statistic.cu): (a) cov of 4 fp32 columns, no binby, 16 B/row; (b) the same on a 128^2 grid over two
            # more fp32 columns, 24 B/row, a 5.2 MB reference grid of 40 fields; (c) OP_MIN_MAX of one fp64 column against b200_minmax
            import ctypes as C
            import subprocess
            from vaex_b200 import statistic as ST
            power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
            cols = [torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen) for _ in range(6)]
            for name, binby, sizes, bpr in (("CV-a", [], [], 16), ("CV-b", cols[4:], [128, 128], 24)):
                st = ST.Statistic(ST.OP_COV.code, _lib.F32, sizes, [-3.0] * len(sizes), [3.0] * len(sizes), False, 4, 1, ctx=ctx)
                ms = timed(lambda: st.bin(0, binby, cols[:4], [None], n, 0), args.reps, setup=st.reset)
                report(name, "cov of 4 fp32 columns" + (" binby 2-D 128^2" if binby else ", no binby"), n, bpr, ms, gpu=power)
                st.close()
            del cols
            torch.cuda.empty_cache()
            x = torch.empty(n, dtype=torch.float64, device="cuda").normal_(generator=gen)
            st = ST.Statistic(ST.OP_MIN_MAX.code, _lib.F64, [], [], [], False, 1, 1, ctx=ctx)
            ms = timed(lambda: st.bin(0, [], [x], [None], n, 0), args.reps, setup=st.reset)
            report("CV-c", "legacy OP_MIN_MAX of one fp64 column (k_stat_reg)", n, 8, ms, gpu=power)
            st.close()
            out = (C.c_double * 2)()
            c = _lib.column(x)
            ms = timed(lambda: _lib.check(_lib.lib().b200_minmax(ctx._h, 0, c.code, c.byteswap, c.ptr, None, c.length, c.memspace, out)), args.reps)
            report("CV-c-minmax", "b200_minmax of the same column", n, 8, ms, gpu=power)
            del x
        elif cfg in ("C5", "C2"):
            x = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
            y = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
            bx = superagg.BinnerScalar_float32(1, "x", -3.0, 3.0, 1024)
            by = superagg.BinnerScalar_float32(1, "y", -3.0, 3.0, 1024)
            g = superagg.Grid([bx, by])
            bx.set_data(0, x)
            by.set_data(0, y)
            if cfg == "C5":
                a = superagg.AggCount_int64(g, 1, 1)

                def run():
                    a.reset(0)
                    g.bin(0, [a], n)
                ms = timed(run, args.reps)
                assert int(a.get_result().sum()) == n
                report("C5/headline", "df.count(binby=[x,y], shape=1024) on fp32 rows, one GPU's shard", n, 8, ms)
            else:
                z = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
                a = superagg.AggSum_float32(g, 1, 1)
                a.set_data(0, z, 0)

                def run():
                    a.reset(0)
                    g.bin(0, [a], n)
                ms = timed(run, args.reps)
                total = float(a.get_result().sum())
                ref = float(z.double().sum())
                assert abs(total - ref) <= 1e-6 * max(1.0, abs(ref)) + 1e-6 * n ** 0.5, (total, ref)
                report("C2", "df.sum(z, binby=[x,y], shape=1024) on fp32 rows", n, 12, ms)
                del z
            del x, y
        elif cfg == "C3":
            cols = [torch.empty(n, dtype=torch.float64, device="cuda").normal_(generator=gen) for _ in range(4)]
            bs = [superagg.BinnerScalar_float64(1, "xyz"[i], -3.0, 3.0, 256) for i in range(3)]
            g = superagg.Grid(bs)
            for b, c in zip(bs, cols):
                b.set_data(0, c)
            aggs = [superagg.AggCount_float64(g, 1, 1), superagg.AggSum_float64(g, 1, 1), superagg.AggSumMoment_float64(g, 1, 1, 2)]
            for a in aggs:
                a.set_data(0, cols[3], 0)

            def run():
                for a in aggs:
                    a.reset(0)
                g.bin(0, aggs, n)
            ms = timed(run, max(2, args.reps // 2))
            assert int(aggs[0].get_result().sum()) == n
            report("C3", "df.mean(v)+df.std(v) (count, sum, sum^2 fused) binby=[x,y,z], shape=256 on fp64 rows", n, 32, ms, grid_cells=len(g))
            del cols
        elif cfg == "C4":
            keys = torch.randint(0, 1_000_000, (n,), device="cuda", dtype=torch.int64, generator=gen) * 256 + 5
            v = torch.empty(n, dtype=torch.float64, device="cuda").normal_(generator=gen)
            torch.cuda.synchronize()  # data generation is asynchronous: keep it out of the timed region
            t0 = time.perf_counter()
            s = superutils.ordered_set_int64(7)
            s.update(keys, -1)
            nkeys = len(s)
            ctx.sync()
            t_pass1 = time.perf_counter() - t0
            # timed again on a warm (already grown) table
            t0 = time.perf_counter()
            s2 = superutils.ordered_set_int64(7)
            s2.update(keys, -1)
            assert len(s2) == nkeys
            t_pass1b = time.perf_counter() - t0
            hb = superagg.BinnerHash_int64(1, "k", s)
            g = superagg.Grid([hb])
            hb.set_data(0, keys)
            asum = superagg.AggSum_float64(g, 1, 1)
            acnt = superagg.AggCount_float64(g, 1, 1)
            for a in (asum, acnt):
                a.set_data(0, v, 0)

            def run():
                asum.reset(0)
                acnt.reset(0)
                g.bin(0, [asum, acnt], n)
            ms2 = timed(run, max(2, args.reps // 2))
            assert int(acnt.get_result().sum()) == n
            report("C4/pass1", "ordered_set_int64.update over 1e6 sparse keys (first build incl. table growth)", n, 8, t_pass1 * 1e3, unique_keys=nkeys,
                   second_build_ms=t_pass1b * 1e3)
            report("C4/pass2", "groupby sum+count through the fused hash binner (probe + 2 REDs per row)", n, 16, ms2, unique_keys=nkeys)
            report("C4/total", "df.groupby(k).agg({v:[sum,count]}) both passes", n, 24, t_pass1b * 1e3 + ms2, unique_keys=nkeys)
            del keys, v
        elif cfg == "NU":
            # per-cell nunique (SURVEY 8f row 3): 64 cells, values drawn from 1e5 / 1e7 distinct ints -> 5e6 / ~1e8-pair tables
            for card in (100_000, 10_000_000):
                gcol = torch.randint(0, 64, (n,), device="cuda", dtype=torch.int32, generator=gen)
                v = torch.randint(0, card, (n,), device="cuda", dtype=torch.int64, generator=gen)
                torch.cuda.synchronize()
                bo = superagg.BinnerOrdinal_int32(1, "g", 64, 0, False, False)
                g = superagg.Grid([bo])
                bo.set_data(0, gcol)
                a = superagg.AggNUnique_int64(g, 1, 1, False, False)
                a.set_data(0, v, 0)
                t0 = time.perf_counter()
                g.bin(0, [a], n)
                ctx.sync()
                t_first = time.perf_counter() - t0
                pairs = int(a.get_result().sum())
                t0 = time.perf_counter()
                g.bin(0, [a], n)  # same rows again: every pair is found, nothing is inserted, the table does not grow
                ctx.sync()
                t_again = time.perf_counter() - t0
                assert int(a.get_result().sum()) == pairs
                report(f"NU/{card}", "nunique(v) binby 64 ordinal cells, int64 values (first pass incl. table growth; second pass = lookups only)", n, 12,
                       t_first * 1e3, distinct_pairs=pairs, lookups_only_ms=t_again * 1e3)
                del gcol, v, a
        elif cfg == "SG":
            # sparse two-key groupby (SURVEY 8f row 4): 3000 x 3000 possible combinations, sum + count of v
            from vaex_b200.frame import Frame
            k1 = torch.randint(0, 3000, (n,), device="cuda", dtype=torch.int64, generator=gen) * 1000 + 7
            k2 = torch.randint(0, 3000, (n,), device="cuda", dtype=torch.int64, generator=gen)
            v = torch.empty(n, dtype=torch.float64, device="cuda").normal_(generator=gen)
            torch.cuda.synchronize()
            df = Frame(dict(k1=k1, k2=k2, v=v))
            t0 = time.perf_counter()
            gb = df.groupby(["k1", "k2"], combine=True)
            ctx.sync()
            t_keys = time.perf_counter() - t0
            t0 = time.perf_counter()
            out = gb.agg({"v": ["sum", "count"]})
            t_agg = time.perf_counter() - t0
            assert int(out["count"].sum()) == n
            report("SG", "df.groupby([k1,k2], combine=True).agg({v:[sum,count]}): 2 key sets + combined-code set, then fused probe pass", n, 24 + 24,
                   (t_keys + t_agg) * 1e3, groups=len(out["count"]), key_sets_ms=t_keys * 1e3, aggregate_ms=t_agg * 1e3)
            del k1, k2, v
        elif cfg == "LS":
            ls_string_list(args, ctx, stream, gen, report)


def ls_string_list(args, ctx, stream, gen, report):
    """LS: df.list(s, binby=g) over 1e8 device-resident strings of 1-32 bytes drawn from a 10^4-word vocabulary, 1e5 ordinal groups
    (AggList_string_int64, csrc/list.cu).  The append pass (one bin() call), the finish on the device (sort + gather) and the D2H of
    the arrow buffers are timed separately with CUDA events on the library's stream; the best of --reps rounds is reported."""
    import numpy as np
    import torch
    from vaex_b200 import superagg
    n, groups, vocab = 100_000_000, 100_000, 10_000
    vlen = torch.randint(1, 33, (vocab,), device="cuda", generator=gen)
    word = torch.randint(0, vocab, (n,), device="cuda", generator=gen)
    lengths = vlen[word]
    offsets = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lengths, 0, out=offsets[1:])
    nbytes = int(offsets[-1])
    data = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    step = 10_000_000
    for r0 in range(0, n, step):  # byte p of a row's string = 'a' + (word * 7 + p) % 26: equal words give equal strings
        r1 = min(r0 + step, n)
        b0, b1 = int(offsets[r0]), int(offsets[r1])
        row = torch.repeat_interleave(torch.arange(r0, r1, device="cuda"), lengths[r0:r1])
        pos = torch.arange(b0, b1, device="cuda") - offsets[row]
        data[b0:b1] = (97 + (word[row] * 7 + pos) % 26).to(torch.uint8)
        del row, pos
    keys = torch.randint(0, groups, (n,), device="cuda", dtype=torch.int32, generator=gen)
    torch.cuda.synchronize()
    b = superagg.BinnerOrdinal_int32(1, "g", groups, 0, False, False)
    g = superagg.Grid([b])
    a = superagg.AggList_string_int64(g, 1, 1)
    b.set_data(0, keys)
    a.set_buffers(0, offsets, data)
    import ctypes as C
    from vaex_b200 import _lib
    L = _lib.lib()
    cells = len(g)
    lo, so, va = np.empty(cells + 1, np.int64), np.empty(n + 1, np.int64), np.empty(n, np.uint8)
    by = np.empty(nbytes, np.uint8)
    for arr in (lo, so, va, by):  # fault the host pages in once, outside the timed copies
        arr.fill(0)
    best = {}
    for rep in range(args.reps + 1):  # round 0 warms up (pool and record arrays grow to size there)
        a.reset(0)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        e[0].record(stream)
        g.bin(0, [a], n)
        e[1].record(stream)
        total, nb = C.c_int64(0), C.c_int64(0)
        _lib.check(L.b200_agg_list_finish(a._h, C.byref(total)))  # sort + count + length scan + gather, on the same stream
        _lib.check(L.b200_agg_list_string_bytes(a._h, C.byref(nb)))
        e[2].record(stream)
        _lib.check(L.b200_agg_list_string_read(a._h, lo.ctypes.data, so.ctypes.data, by.ctypes.data, va.ctypes.data))
        e[3].record(stream)
        ctx.sync()
        torch.cuda.synchronize()
        assert total.value == n and nb.value == nbytes
        if rep:
            for k, (i, j) in dict(append=(0, 1), finish=(1, 2), d2h=(2, 3)).items():
                best[k] = min(best.get(k, float("inf")), e[i].elapsed_time(e[j]))
    assert lo[-1] == n and so[-1] == nbytes and va.all()
    best_append = best["append"]
    mean = nbytes / n
    radix_passes = 3  # keys < 2^17 (groups + 2 cells): three 8-bit passes
    # algorithmic bytes per row.  append: key 4 + offsets 8 read, string read + written to the pool, key/payload/start 24 written.
    # finish: per radix pass key + payload read and written (32), the count pass reads keys (8), lengths read payload + two starts
    # and write the length (32), the int64 scan reads + writes it twice (32), the gather reads payload, start, two offsets and the
    # string and writes the string and a validity byte (33 + 2 * mean); the D2H (into pageable numpy memory whose pages are already
    # faulted in) moves the string offsets, bytes and validity (9 + mean) over PCIe, so its rate is not an HBM figure
    append_bpr = 4 + 8 + 2 * mean + 24
    finish_bpr = 32 * radix_passes + 8 + 32 + 32 + 33 + 2 * mean
    d2h_bpr = 9 + mean
    report("LS/append", "AggList_string_int64 append: one bin() call over 1e8 device strings of 1-32 B, 1e5 ordinal groups", n, append_bpr, best_append,
           string_bytes=nbytes, mean_string_bytes=mean)
    report("LS/finish", "AggList_string_int64 finish on the device: radix sort by cell + per-cell count + int64 length scan + byte gather", n,
           finish_bpr, best["finish"], string_bytes=nbytes, radix_passes=radix_passes)
    report("LS/d2h", "AggList_string_int64 read: D2H of the arrow buffers into pageable numpy arrays", n, d2h_bpr, best["d2h"], string_bytes=nbytes)
    report("LS/finish+d2h", "AggList_string_int64 result: finish + D2H", n, finish_bpr + d2h_bpr, best["finish"] + best["d2h"], string_bytes=nbytes)
    del offsets, data, keys, word, lengths


if __name__ == "__main__":
    main()
