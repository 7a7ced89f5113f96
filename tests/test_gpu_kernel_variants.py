"""Every binned-aggregation kernel variant on the edge-value corpus, with proof of which kernel ran.

`launch_binby` (csrc/binby.cu) picks a kernel from the row count, the grid's bytes, dtypes, masks and alignment.  Each case here
builds a problem that selects one variant, records the kernels the call launched with torch.profiler, asserts the intended one
is among them, and compares the grids with the oracle bit for bit, or with exact arithmetic where DESIGN §3 says bits cannot
match (helpers.check_exact).  A threshold that moves makes these tests fail instead of silently moving coverage.
"""
import re
from fractions import Fraction

import numpy as np
import pytest

import golden_util
from helpers import B200Binby, check_exact, edge_column, gamma, random_case, same_bits

pytestmark = pytest.mark.gpu

VALUE_DTYPES = ["f8", "f4", "i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?", ">f8", ">i4", ">u2"]


def launched(fn):
    """(fn(), the names of the CUDA kernels it launched); fails when the profiler saw no kernel at all.  The profiler now and then
    returns a session without its kernel records, so `fn` must be repeatable: it is run a second time when that happens."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(2):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset"))}
        if names:
            return out, names
    raise AssertionError("torch.profiler recorded no CUDA kernel")


def assert_ran(names, pattern):
    assert any(re.search(pattern, n) for n in names), (pattern, sorted(names))


def run(binners, aggs, n, start=0, chunk=None, nthreads=1, device="resident"):
    return launched(lambda: B200Binby(binners, aggs, nthreads).run(n, chunk, device, start=start))


def tail(specs, start):
    """the same specs restricted to rows [start:] (what the oracle sees of a run that starts at `start`)"""
    out = []
    for s in specs:
        s = dict(s)
        for k in ("data", "mask", "order", "selection"):
            if s.get(k) is not None:
                s[k] = s[k][start:]
        out.append(s)
    return out


def generic_aggs(O, rng, v, n, moment):
    mask = (rng.random(n) < 0.8).astype("u1")
    return [O.agg("count", None, mask), O.agg("count", v), O.agg("sum", v), O.agg("sum_moment", v, mask, moment=moment),
            O.agg("min", v, mask), O.agg("max", v)]


# k_binby<VEC, SMEM>: integer (ordinal) keys keep fast.cu out; small grid + >= 4096 rows -> shared-memory copies; n < 4096 or a
# grid over 96 KB -> global REDs; a start off the 16-byte boundary -> scalar loads
GENERIC = {  # name: (rows, ordinal count, start, chunk, kernel)
    "vec_global_small_n": (3000, 7, 0, None, r"k_binby<true, false>"),
    "vec_global_big_grid": (20000, 9000, 0, None, r"k_binby<true, false>"),
    "vec_smem": (20000, 7, 0, None, r"k_binby<true, true>"),
    "scalar_global": (9001, 7, 1, 1001, r"k_binby<false, false>"),
    "scalar_smem": (20001, 7, 1, 4099, r"k_binby<false, true>"),
}


@pytest.mark.parametrize("variant", sorted(GENERIC))
def test_generic_kernel(variant, oracle):
    n, count, start, chunk, kernel = GENERIC[variant]
    rng = np.random.default_rng(40 + sorted(GENERIC).index(variant))
    key = rng.integers(-1, count + 1, n).astype("i4")
    binners = [oracle.ordinal(key, count, 0, True, False)]
    problems = [generic_aggs(oracle, rng, edge_column(rng, dt, n), n, moment=j % 9) for j, dt in enumerate(VALUE_DTYPES)]
    gots, names = launched(lambda: [B200Binby(binners, aggs, 3 if chunk else 1).run(n, chunk, "resident", start=start) for aggs in problems])
    assert_ran(names, kernel)
    b = tail(binners, start)
    for dt, aggs, got in zip(VALUE_DTYPES, problems, gots):
        a = tail(aggs, start)
        check_exact(b, a, n - start, oracle.binby(b, a, n - start), got, (variant, dt))


# k_binby_fast (csrc/fast.cu): float keys of one width, no masks, count* / count / sum / sum^2 of one float column, >= 8192 rows;
# all accumulators of a copy within 96 KB -> shared-memory copies, else global REDs
@pytest.mark.parametrize("smem", [True, False])
@pytest.mark.parametrize("kdt", ["f4", "f8"])
@pytest.mark.parametrize("vdt", ["f4", "f8"])
def test_fast_kernel(kdt, vdt, smem, oracle):
    rng = np.random.default_rng(50 + 4 * (kdt == "f8") + 2 * (vdt == "f8") + smem)
    n = 30011
    bins = (10, 6) if smem else (4000, 3)  # 13 x 9 cells vs 4003 x 6 cells x 24 B > 96 KB
    keys = [edge_column(rng, kdt, n, scale=2.0) for _ in bins]
    v = edge_column(rng, vdt, n)
    binners = [oracle.scalar(k, -2.5, 3.1, b) for k, b in zip(keys, bins)]
    aggs = [oracle.agg("count"), oracle.agg("count", v), oracle.agg("sum", v), oracle.agg("sum_moment", v, moment=2)]
    got, names = run(binners, aggs, n)
    T, TV = ("float" if kdt == "f4" else "double"), ("float" if vdt == "f4" else "double")
    assert_ran(names, rf"k_binby_fast<{T}, 2, {TV}, true, {'true' if smem else 'false'}>")
    check_exact(binners, aggs, n, oracle.binby(binners, aggs, n), got, (kdt, vdt, smem))


def test_region_sorted_kernels(oracle, monkeypatch):
    """csrc/tilesort.cu, forced on a small problem through its per-call knobs"""
    monkeypatch.setenv("B200_TILESORT_FORCE", "1")
    monkeypatch.setenv("B200_TILESORT_MIN_ROWS", "1000")
    rng = np.random.default_rng(61)
    n = 100_003
    for kdt, vdt in (("f4", "f8"), ("f8", "f4")):
        keys = [edge_column(rng, kdt, n, scale=2.0) for _ in range(2)]
        v = edge_column(rng, vdt, n)
        binners = [oracle.scalar(k, -3, 3, 300) for k in keys]
        aggs = [oracle.agg("count"), oracle.agg("count", v), oracle.agg("sum", v), oracle.agg("sum_moment", v, moment=2)]
        got, names = run(binners, aggs, n)
        assert_ran(names, r"k_sort_partition")
        assert_ran(names, r"k_sort_apply")
        check_exact(binners, aggs, n, oracle.binby(binners, aggs, n), got, (kdt, vdt))


def test_ring_partition_fp64_edge_keys(oracle):
    """csrc/ringcount.cu with float64 keys from the edge corpus: subnormals, +-inf, NaN payloads, keys on / next to bin edges"""
    rng = np.random.default_rng(62)
    n = (1 << 22) + 4097
    bins = (700, 900)
    keys = []
    for b in bins:
        e = -3 + 6 * np.arange(b + 1) / b
        k = edge_column(rng, "f8", n, scale=1.0)
        at = rng.random(n) < 0.1
        k[at] = rng.choice(np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf)]), int(at.sum()))
        keys.append(k)
    binners = [oracle.scalar(k, -3, 3, b) for k, b in zip(keys, bins)]
    got, names = run(binners, [oracle.agg("count")], n)
    assert_ran(names, r"k_ring_partition<double")
    assert_ran(names, r"k_ring_count")
    assert same_bits(oracle.binby(binners, [oracle.agg("count")], n)[0], got[0]) and int(got[0].sum()) == n


ORDER_DTYPES = ["f8", "f4", "i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1"]


@pytest.mark.parametrize("vec", [True, False])
def test_first_last_kernels(vec, oracle):
    """csrc/first.cu with every order dtype (edge values: +-0.0 ties, -inf, INT64_MIN, NaN orders skipped), chunked over three
    slots (vector loads from row 0, scalar loads from an odd row); no order column and a mask past 1024 rows in one call"""
    rng = np.random.default_rng(70 + vec)
    n = 5003
    start, chunk = (0, 2048) if vec else (1, 1777)
    key = rng.integers(0, 6, n).astype("i2")
    binners = [oracle.ordinal(key, 5, 0, True)]
    problems = []
    for odt in ORDER_DTYPES:
        v = edge_column(rng, "f8" if odt[-1] in "48" else "i2", n)
        order = edge_column(rng, odt, n)
        if np.dtype(odt).kind == "f":  # many ties between +0.0 and -0.0
            at = rng.random(n) < 0.1
            order[at] = np.where(rng.random(int(at.sum())) < 0.5, 0.0, -0.0)
        problems.append([oracle.agg("first", v, None, order=order), oracle.agg("last", v, None, order=order)])
    gots, names = launched(lambda: [B200Binby(binners, aggs, 3).run(n, chunk, "resident", start=start) for aggs in problems])
    assert_ran(names, rf"k_first_select<{'true' if vec else 'false'}>")
    b = tail(binners, start)
    for odt, aggs, got in zip(ORDER_DTYPES, problems, gots):
        for w, g in zip(oracle.binby(b, tail(aggs, start), n - start), got):
            assert same_bits(w, g), odt
    v = edge_column(rng, ">f8", n)
    mask = (rng.random(n) < 0.6).astype("u1")
    aggs = [oracle.agg("first", v, mask), oracle.agg("last", v, mask)]
    got, names = run(binners, aggs, n, start=start)
    assert_ran(names, rf"k_first_select<{'true' if vec else 'false'}>")
    b, a = tail(binners, start), tail(aggs, start)
    for w, g in zip(oracle.binby(b, a, n - start), got):
        assert same_bits(w, g)


def test_nunique_edges_chunked(oracle):
    """csrc/nunique.cu on edge values (+-0.0 are two keys, every NaN payload is one nan), selections, dropmissing / dropnan, over
    three calls on three slots"""
    rng = np.random.default_rng(80)
    n = 9001
    key = rng.integers(0, 4, n).astype("u1")
    binners = [oracle.ordinal(key, 4)]
    problems = []
    for dt in VALUE_DTYPES:
        v = edge_column(rng, dt, n)
        valid = (rng.random(n) < 0.9).astype("u1")
        sel = (rng.random(n) < 0.8).astype("u1")
        problems.append([oracle.agg("nunique", v), oracle.agg("nunique", v, valid, selection=sel, dropmissing=True),
                         oracle.agg("nunique", v, valid, dropnan=True)])
    gots, names = launched(lambda: [B200Binby(binners, aggs, 3).run(n, 3001, "resident", start=1) for aggs in problems])
    assert_ran(names, r"k_nunique<false>")
    for dt, aggs, got in zip(VALUE_DTYPES, problems, gots):
        for w, g in zip(oracle.binby(tail(binners, 1), tail(aggs, 1), n - 1), got):
            assert same_bits(w, g), dt


def test_nunique_table_grows_between_calls():
    """more than 5e6 distinct (cell, value) pairs over three calls: the table is rehashed while it holds earlier calls' keys"""
    import torch
    from vaex_b200 import superagg
    n = 6_000_000
    i = torch.arange(n, device="cuda", dtype=torch.int64)
    key = (i % 5).to(torch.int32)
    v = (i // 2).to(torch.float64)  # every value twice: once in an even, once in an odd cell of the pair
    v[::1001] = -0.0
    v[::1003] = 0.0
    v[::997] = float("nan")
    b = superagg.BinnerOrdinal_int32(1, "k", 5, 0, False, False)
    grid = superagg.Grid([b])

    def go():
        agg = superagg.AggNUnique_float64(grid, 1, 1, False, False)
        for lo, hi in ((0, 2_000_001), (2_000_001, 4_000_000), (4_000_000, n)):
            b.set_data(0, key[lo:hi])
            agg.set_data(0, v[lo:hi], 0)
            agg.clear_data_mask(0)
            agg.clear_selection_mask(0)
            grid.bin(0, [agg], hi - lo)
        return agg.get_result()
    got, names = launched(go)
    assert_ran(names, r"k_nunique_rehash")
    kh, vh = key.cpu().numpy(), v.cpu().numpy()
    nan = np.isnan(vh)
    want = [np.unique(vh[(kh == c) & ~nan].view(np.int64)).size + int(((kh == c) & nan).any()) for c in range(5)] + [0, 0]
    assert got.tolist() == want


# ---- heavy cells ---------------------------------------------------------------------------------------------------------------
def test_heavy_cells_through_both_smem_kernels():
    """1e8 rows into 13 (fast.cu) and 16 (k_binby) cells: the private shared-memory sums and their flush.  Integer-valued floats
    sum exactly, so those sums are bit-exact; a cancelling column (+-1e8 plus dyadic residuals) is held to the recursive-summation
    bound of its exact sum; integer sums and counts are exact."""
    import torch
    from vaex_b200 import superagg
    n = 100_000_000
    i = torch.arange(n, device="cuda", dtype=torch.int64)
    r = i % 1024
    canc = torch.where(i % 2 == 0, 1e8, -1e8).to(torch.float64) + r.to(torch.float64) / 1024  # exact in float64
    small = ((i % 7) - 3).to(torch.float32)
    for C, fast in ((13, True), (16, False)):
        cell = i % C
        if fast:
            bx = superagg.BinnerScalar_float32(1, "x", 0, C, C)
            bx.set_data(0, cell.to(torch.float32) + 0.5)
        else:
            bx = superagg.BinnerOrdinal_int32(1, "x", C, 0, False, False)
            bx.set_data(0, cell.to(torch.int32))
        grid = superagg.Grid([bx])
        if fast:
            specs = [("AggCount_int64", None), ("AggCount_float32", small), ("AggSum_float32", small), ("AggSumMoment_float32", small)]
        else:
            specs = [("AggCount_int64", None), ("AggSum_float64", canc), ("AggSum_int64", i), ("AggMax_float64", canc)]

        def go(specs=specs, grid=grid):
            aggs = []
            for cls, col in specs:
                a = getattr(superagg, cls)(grid, 1, 1, 2) if "Moment" in cls else getattr(superagg, cls)(grid, 1, 1)
                if col is not None:
                    a.set_data(0, col, 0)
                a.clear_data_mask(0)
                aggs.append(a)
            grid.bin(0, aggs, n)
            return [a.get_result() for a in aggs]
        got, names = launched(go)
        inner = slice(2, C + 2) if fast else slice(0, C)
        counts = torch.bincount(cell, minlength=C).cpu().numpy()
        assert got[0][inner].tolist() == counts.tolist() and got[0].sum() == n
        if fast:
            assert_ran(names, r"k_binby_fast<float, 1, float, true, true>")
            s = small.double()
            assert got[1][inner].tolist() == counts.tolist()
            assert got[2][inner].tolist() == torch.zeros(C, dtype=torch.float64, device="cuda").index_add_(0, cell, s).cpu().tolist()
            assert got[3][inner].tolist() == torch.zeros(C, dtype=torch.float64, device="cuda").index_add_(0, cell, s * s).cpu().tolist()
            # the same column as the cancelling float64 values through the fast kernel's float64 accumulators
            got2, names2 = launched(lambda: go([("AggSum_float64", canc)])[0])
            assert_ran(names2, r"k_binby_fast<float, 1, double, true, true>")
            cancel = got2[inner]
        else:
            assert_ran(names, r"k_binby<true, true>")
            isum = torch.zeros(C, dtype=torch.int64, device="cuda").index_add_(0, cell, i).cpu().numpy()
            assert same_bits(got[2][inner], isum)
            # cell c holds the rows i = c (mod 16): one sign, residuals r = i % 1024 = c (mod 16), the largest 1008 + c
            assert got[3][inner].tolist() == [(1e8 if c % 2 == 0 else -1e8) + (1008 + c) / 1024 for c in range(C)]
            cancel = got[1][inner]
        # exact sums: sum of residuals in 1/1024 units minus the +-1e8 that cancel (even cells of an odd C see both signs)
        sign = torch.where(i % 2 == 0, 1, -1)
        units = torch.zeros(C, dtype=torch.int64, device="cuda").index_add_(0, cell, sign * (100_000_000 * 1024) + r).cpu().tolist()
        k = counts.tolist()
        for c in range(C):
            exact, mag = Fraction(units[c], 1024), k[c] * Fraction(10 ** 8 + 1)  # mag >= sum |x_i|
            assert abs(Fraction(float(cancel[c])) - exact) <= Fraction(gamma(k[c])) * mag, (C, c, float(cancel[c]), float(exact))


def test_count_cell_past_2p32():
    """one cell counted past 2^32 by three bin() calls over the same 1.5e9-row device column"""
    import torch
    from vaex_b200 import superagg
    n = 1_500_000_000
    x = torch.zeros(n, dtype=torch.uint8, device="cuda")
    b = superagg.BinnerOrdinal_uint8(1, "x", 1, 0, False, False)
    grid = superagg.Grid([b])
    b.set_data(0, x)

    def go():
        agg = superagg.AggCount_int64(grid, 1, 1)
        agg.clear_data_mask(0)
        for _ in range(3):
            grid.bin(0, [agg], n)
        return agg.get_result()
    got, names = launched(go)
    assert_ran(names, r"k_binby<true, true>")
    assert got.tolist() == [3 * n, 0, 0]


# ---- the edge corpus through whatever kernel it selects, and the golden edge cases ------------------------------------------
@pytest.mark.parametrize("seed", range(16))
def test_edge_corpus_random(seed, oracle):
    rng = np.random.default_rng(8000 + seed)
    n = int(rng.integers(1, 12000))
    binners, aggs = random_case(rng, n, edges=True)
    want = oracle.binby(binners, aggs, n)
    for device, chunk, nthreads in ((False, None, 1), ("resident", None, 1), ("resident", 1001, 3)):
        if chunk and any(a["op"] in ("first", "last") and (a["mask"] is not None or a["order"] is None) for a in aggs):
            continue  # first/last judge the mask and, without an order column, order by row inside each call: one call only
        got = B200Binby(binners, aggs, nthreads).run(n, chunk, device)
        check_exact(binners, aggs, n, want, got, (device, chunk))


EDGES = golden_util.load_edges()


@pytest.mark.parametrize("name", sorted(EDGES))
def test_golden_edges(name, oracle):
    binners, aggs, n, expected = golden_util.binby_case(EDGES[name])
    got = B200Binby(binners, aggs).run(n, None, "resident")
    check_exact(binners, aggs, n, expected, got, name)


def test_integer_moment_known_answers(oracle):
    """the reference's out-of-range conversion per row (int64 -> INT64_MIN, uint64 >= 2^64 -> 0); past 2^53 the device's rule: the
    exact sum of the converted powers (DESIGN §3), which here differs from the reference's double-rounded running sum"""
    from helpers import int_moment_rule
    for name, want in (("kat_moment3_int64_out_of_range", np.iinfo(np.int64).min), ("kat_moment3_uint64_out_of_range", 0)):
        binners, aggs, n, expected = golden_util.binby_case(EDGES[name])
        got = B200Binby(binners, aggs).run(n)
        assert got[0].ravel()[2] == want and same_bits(got[0], expected[0]), name
    binners, aggs, n, expected = golden_util.binby_case(EDGES["kat_moment4_past_2p53"])
    got = B200Binby(binners, aggs).run(n)
    rule, exact = int_moment_rule(binners, aggs[0], n)
    assert not exact.ravel()[2] and same_bits(got[0], rule)
    assert int(got[0].ravel()[2]) == sum(int(float(x) ** 4) for x in (30000, 30001, 29999, 1))
    assert int(expected[0].ravel()[2]) == 2430000010800000000 != int(got[0].ravel()[2])


def test_signed_zero_min_max_rule(oracle):
    """min over both zeros is -0.0 and max is +0.0 whatever the arrival order (DESIGN §3); the reference keeps the last arrival"""
    for v in (np.array([0.0, -0.0]), np.array([-0.0, 0.0]), np.array([0.0, -0.0], "f4"), np.array([-0.0, 0.0, -0.0], ">f8")):
        b = [oracle.scalar(np.full(len(v), 0.5), 0, 1, 1)]
        got = B200Binby(b, [oracle.agg("min", v), oracle.agg("max", v)]).run(len(v))
        assert np.signbit(got[0].ravel()[2]) and not np.signbit(got[1].ravel()[2]), v
    binners, aggs, n, expected = golden_util.binby_case(EDGES["kat_minmax_signed_zeros"])
    assert np.signbit(expected[0].ravel()[2]) and np.signbit(expected[1].ravel()[2])  # the reference: the last-arriving -0.0
