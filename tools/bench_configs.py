#!/usr/bin/env python
"""Times every BASELINE.json configuration on one H100 with device-resident columns (the roofline setting) and prints one
JSON object per config: rows/s, achieved algorithmic GB/s (SURVEY.md 8d bytes/row) and the fraction of the measured HBM peak.

    python tools/bench_configs.py [--rows 1e9] [--configs C1,C2,C3,C4,C5,CV,PA,MI,MO]

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
        elif cfg == "PA":
            pa_percentile(args, n, ctx, stream, gen, timed, report)
        elif cfg == "MI":
            mi_mutual_information(args, n, ctx, stream, gen, timed, report)
        elif cfg == "MO":
            mo_mode(args, n, ctx, stream, gen, timed, report)


def pa_percentile(args, n, ctx, stream, gen, timed, report):
    """PA: df.percentile_approx(z, [25, 50, 75]) over `n` device-resident fp32 rows, (a) binby=[x, y] 128^2 in [-3, 3] with 1024
    percentile bins in [-4, 4] (a 131^2 x 1027 int64 grid, 141 MB: k_pct_cell) and (b) no binby with 65536 percentile bins (one cell:
    k_pct_block).  Timed separately with CUDA events: the count pass and the device finish (b200_grid_percentile).  Beside them the host
    finish the reference runs: the D2H of the count grid into pageable memory and the vectorised numpy restatement of the finish
    (tests/percentile_oracle.py), which is a lower bound of the reference's own, whose index_choose loops over every cell in Python."""
    import subprocess
    import numpy as np
    import torch
    from vaex_b200 import percentile as _pct, superagg
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import percentile_oracle as PO
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cols = [torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen) for _ in range(3)]
    pct = [25, 50, 75]
    for name, nd, P in (("PA-2d", 2, 1024), ("PA-none", 0, 65536)):
        bs = [superagg.BinnerScalar_float32(1, "xy"[i], -3.0, 3.0, 128) for i in range(nd)] + [superagg.BinnerScalar_float32(1, "z", -4.0, 4.0, P)]
        g = superagg.Grid(bs)
        for b, c in zip(bs, cols[2 - nd:]):
            b.set_data(0, c)
        a = superagg.AggCount_int64(g, 1, 1)

        def count():
            a.reset(0)
            g.bin(0, [a], n)
        ms_count = timed(count, args.reps)
        ptr, nbytes = a.device_pointer(0)
        cells = int(np.prod([s - 3 for s in g.shapes[:-1]], dtype=np.int64))
        out = torch.empty((len(pct), cells), dtype=torch.float64, device="cuda")
        ms_finish = timed(lambda: _pct.grid_percentile(ptr, g.shapes, -4.0, 8.0, pct, ctx=ctx, out=out), args.reps)
        host_best = d2h_best = None
        for _ in range(max(2, args.reps // 2)):
            t0 = time.perf_counter()
            grid = a.get_result()  # D2H into pageable memory
            t1 = time.perf_counter()
            want = PO.percentile_approx([grid], [[-4, 4]], pct, False)
            t2 = time.perf_counter()
            d2h_best = min(d2h_best or 1e30, (t1 - t0) * 1e3)
            host_best = min(host_best or 1e30, (t2 - t0) * 1e3)
        got = out.cpu().numpy().reshape((len(pct),) + tuple(s - 3 for s in g.shapes[:-1]), order="F")
        assert int(grid.sum()) == n and np.array_equal(got.view(np.int64), np.asarray(want).reshape(got.shape).view(np.int64))
        workload = "percentile_approx(z, [25, 50, 75]" + (", binby=[x, y] shape 128" if nd else "") + f", percentile_shape={P}) on fp32 rows"
        report(name + "/count", workload + ": count pass", n, 4 * (nd + 1), ms_count, gpu=power)
        print(json.dumps(dict(config=name + "/finish", workload=workload + ": finish on the device", kernel="k_pct_cell" if cells >= 2048 else "k_pct_block",
                              ms=ms_finish, grid_bytes=nbytes, grid_reads_gbs=2 * nbytes / (ms_finish * 1e-3) / 1e9, gpu=power)), flush=True)
        print(json.dumps(dict(config=name + "/host_finish", workload=workload + ": D2H (pageable) + numpy finish on the host", ms=host_best, d2h_ms=d2h_best,
                              grid_bytes=nbytes, gpu=power)), flush=True)
        del a, g, out, grid
        torch.cuda.empty_cache()
    del cols


def mi_mutual_information(args, n, ctx, stream, gen, timed, report):
    """MI: df.mutual_information over `n` device-resident fp32 rows, y correlated with x, mi_shape=256 in [-5, 5]^2.
    MI-pair: (x, y), one cell (a 259^2 int64 grid: the split regime).  MI-binby: the same with binby=[z], shape=128 in [-3, 3]
    (259^2 x 131 int64 = 70 MB, 128 cells: the split regime), the device finish against the host finish the reference runs (D2H of the
    grid into pageable memory + the numpy restatement of tests/mutual_information_oracle.py, a lower bound of the reference's per-cell
    Python loop).  Count pass and finish are timed separately with CUDA events; each finish is checked against the restatement on
    the same grid, within the per-cell bound of DESIGN.md section 3, before the timed runs.  MI-matrix: x=[8 columns] end to end
    through Frame (one minmax pass per column, 36 unique pairs in one executor pass), wall clock; before the timed runs every
    unique entry is checked against the restatement's finish of that pair's count grid."""
    import subprocess
    import numpy as np
    import torch
    from vaex_b200 import execution, frame, superagg
    from vaex_b200 import mutual_information as _mi
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mutual_information_oracle as MO
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    x = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    y = x + torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    z = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    parity = True
    for name, nb in (("MI-pair", 0), ("MI-binby", 1)):
        bs = [superagg.BinnerScalar_float32(1, e, -5.0, 5.0, 256) for e in "xy"] + [superagg.BinnerScalar_float32(1, "z", -3.0, 3.0, 128)][:nb]
        g = superagg.Grid(bs)
        for b, c in zip(bs, (x, y, z)):
            b.set_data(0, c)
        a = superagg.AggCount_int64(g, 1, 1)

        def count():
            a.reset(0)
            g.bin(0, [a], n)
        ms_count = timed(count, args.reps)
        ptr, nbytes = a.device_pointer(0)
        cells = 128 if nb else 1
        out = torch.empty(cells, dtype=torch.float64, device="cuda")
        _mi.grid_mutual_information(ptr, g.shapes, 2, ctx=ctx, out=out)
        grid = a.get_result()[(slice(2, -1),) * (2 + nb)]
        want, tol = (np.array([MO.mi_cell(grid[..., i].astype(np.float64)) for i in range(cells)]), np.array([MO.bound(grid[..., i]) for i in range(cells)])) \
            if nb else (np.array([MO.mi_cell(grid.astype(np.float64))]), np.array([MO.bound(grid)]))
        ok = int(a.get_result().sum()) == n and bool(np.all(np.abs(out.cpu().numpy() - want) <= tol))
        parity &= ok
        ms_finish = timed(lambda: _mi.grid_mutual_information(ptr, g.shapes, 2, ctx=ctx, out=out), args.reps)
        host_best = d2h_best = None
        for _ in range(max(2, args.reps // 2)):
            t0 = time.perf_counter()
            full = a.get_result()  # D2H into pageable memory
            t1 = time.perf_counter()
            MO.calculate(full[(slice(2, -1),) * (2 + nb)], nb)
            t2 = time.perf_counter()
            d2h_best = min(d2h_best or 1e30, (t1 - t0) * 1e3)
            host_best = min(host_best or 1e30, (t2 - t0) * 1e3)
        workload = "mutual_information(x, y, mi_shape=256" + (", binby=[z], shape=128" if nb else "") + ") on fp32 rows"
        report(name + "/count", workload + ": count pass", n, 4 * (2 + nb), ms_count, gpu=power)
        print(json.dumps(dict(config=name + "/finish", workload=workload + ": finish on the device", ms=ms_finish, grid_bytes=nbytes,
                              grid_reads_gbs=2 * nbytes / (ms_finish * 1e-3) / 1e9, parity=ok, gpu=power)), flush=True)
        print(json.dumps(dict(config=name + "/host_finish", workload=workload + ": D2H (pageable) + numpy finish on the host", ms=host_best,
                              d2h_ms=d2h_best, grid_bytes=nbytes, gpu=power)), flush=True)
        del a, g, out, grid, full
        torch.cuda.empty_cache()
    cols = {"x": x, "y": y, "z": z}
    for k in range(5):
        cols[f"c{k}"] = (x if k % 2 else z) * 0.5 + torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    f = frame.Frame(cols, executor=execution.Executor(1))
    names = list(cols)
    # checked before the timed runs: every unique entry against the restatement's finish of that pair's count grid (same limits)
    m = f.mutual_information(names, mi_shape=256)
    limits = {e: list(f.minmax(e)) for e in names}
    ok = m.shape == (8, 8) and np.array_equal(m, m.T)
    for i in range(8):
        for j in range(i, 8):
            counts = f.count(binby=[names[i], names[j]], limits=[limits[names[i]], limits[names[j]]], shape=256)
            ok = ok and bool(abs(m[i, j] - MO.mi_cell(counts.astype(np.float64))) <= MO.bound(counts))
    parity &= ok
    best = None
    for _ in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f.mutual_information(names, mi_shape=256)
        torch.cuda.synchronize()
        best = min(best or 1e30, (time.perf_counter() - t0) * 1e3)
    print(json.dumps(dict(config="MI-matrix", workload="mutual_information(x=[8 fp32 columns], mi_shape=256) end to end: 8 minmax passes (one per "
                          "column), 36 count grids in one pass, 36 device finishes", rows=n, ms=best, parity=ok, gpu=power)), flush=True)
    print(json.dumps(dict(config="MI", parity=bool(parity), gpu=power)), flush=True)
    del f, cols, x, y, z


def mo_mode(args, n, ctx, stream, gen, timed, report):
    """MO: df.mode(v, binby, mode_shape=64, mode_limits=[-4, 4]) over `n` device-resident fp32 rows, (a) binby=[x] shape 256 (a 64 x 256
    grid: the shared-memory count) and (b) binby=[x, y] shape 256 (64 x 256^2 = 4M cells, 32 MB: the global count), limits [-3, 3].
    Timed separately with CUDA events: the count pass and the device finish (b200_stat_mode, which includes copying the modes back).
    Beside them the host finish the reference runs: the D2H of the count grid and numpy's argmax finish (tests/mode_oracle.finish).
    Parity: the device histogram and finish of the first 2^22 rows against the numpy restatement of those rows, bit for bit."""
    import subprocess
    import numpy as np
    import torch
    from vaex_b200 import mode as _mode
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import mode_oracle as MO
    from helpers import same_bits
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    x, y, v = (torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen) for _ in range(3))
    centers = _mode.centers(-4.0, 4.0, 64)
    sub = 1 << 22
    parity = True
    for name, binby in (("MO-1d", [x]), ("MO-2d", [x, y])):
        shape = (64,) + (256,) * len(binby)
        blocks = binby + [v]
        lims = [(-3.0, 3.0)] * len(binby) + [(-4.0, 4.0)]
        order, olims = _mode.axis_order(blocks), _mode.axis_order(lims)
        h = _mode.Histogram(shape, [lo for lo, _ in olims], [hi for _, hi in olims], ctx=ctx)
        small = _mode.Histogram(shape, [lo for lo, _ in olims], [hi for _, hi in olims], ctx=ctx)
        small.bin(0, [c[:sub] for c in order], [], [None], sub, 0)
        got = small.mode(centers)
        small.close()
        want = MO.finish(MO.histogram([c[:sub].cpu().numpy() for c in blocks], lims, shape), -4.0, 4.0, 64)
        ok = same_bits(got, want)
        parity &= ok

        def count():
            h.bin(0, order, [], [None], n, 0)
        ms_count = timed(count, args.reps, setup=h.reset)
        ms_finish = timed(lambda: h.mode(centers), args.reps)
        host_best = d2h_best = None
        for _ in range(max(2, args.reps // 2)):
            t0 = time.perf_counter()
            grid = h.read()  # D2H into pageable memory
            t1 = time.perf_counter()
            MO.finish(grid, -4.0, 4.0, 64)
            t2 = time.perf_counter()
            d2h_best = min(d2h_best or 1e30, (t1 - t0) * 1e3)
            host_best = min(host_best or 1e30, (t2 - t0) * 1e3)
        assert int(grid.sum()) <= n
        workload = f"mode(v, binby=[{', '.join('xy'[:len(binby)])}], shape=256, mode_shape=64) on fp32 rows"
        report(name + "/count", workload + ": count pass", n, 4 * len(blocks), ms_count,
               kernel="k_stat_count_smem" if np.prod(shape) * 4 <= 96 * 1024 else "k_stat_global", gpu=power)
        print(json.dumps(dict(config=name + "/finish", workload=workload + ": argmax finish on the device, modes copied back", ms=ms_finish,
                              grid_bytes=8 * int(np.prod(shape)), parity=ok, gpu=power)), flush=True)
        print(json.dumps(dict(config=name + "/host_finish", workload=workload + ": D2H (pageable) + numpy finish on the host", ms=host_best,
                              d2h_ms=d2h_best, gpu=power)), flush=True)
        h.close()
        del h, grid
        torch.cuda.empty_cache()
    print(json.dumps(dict(config="MO", parity=bool(parity), gpu=power)), flush=True)
    del x, y, v


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
