"""GPU parity: the CUDA path (through the C ABI, via the superagg mirror) against the oracle on identical inputs.

Bar: bit-exact for counts / min / max / first-last / integer sums / bin indices; floating sums and moments within 1e-6
relative (asserted far tighter here because the test grids hold few rows per cell).
"""
import numpy as np
import pytest

from helpers import b200_binby, random_case, same

pytestmark = pytest.mark.gpu

RTOL = 1e-6  # the north-star tolerance for floating-point sums/moments


def check(binners, aggs, n, oracle, **kw):
    want = oracle.binby(binners, aggs, n)
    got = b200_binby(binners, aggs, n, **kw)
    for a, w, g in zip(aggs, want, got):
        is_float_sum = a["op"] in ("sum", "sum_moment") and np.asarray(a["data"]).dtype.kind == "f"
        if is_float_sum:
            scale = max(1.0, float(np.nanmax(np.abs(w)))) if w.size else 1.0
            assert w.shape == g.shape and w.dtype == g.dtype
            assert np.allclose(g, w, rtol=RTOL, atol=1e-9 * scale), (a["op"], a["data"].dtype)
        else:
            assert same(w, g), (a["op"], None if a["data"] is None else a["data"].dtype, [b["kind"] for b in binners])


def test_kat_count_1d(oracle):
    # /root/reference/tests/agg_test.py:150-158
    x = np.array([-1, -2, 0.5, 1.5, 4.5, 5], dtype="f8")
    got = b200_binby([oracle.scalar(x, 0, 5, 5)], [oracle.agg("count")])[0]
    assert got.tolist() == [0, 2, 1, 1, 0, 0, 1, 1]


def test_kat_count_1d_ordinal(oracle):
    # /root/reference/tests/agg_test.py:171-180
    x = np.array([-1, -2, 0, 1, 4, 5], dtype="i8")
    got = b200_binby([oracle.ordinal(x, 5, 0)], [oracle.agg("count")])[0]
    want = oracle.binby([oracle.ordinal(x, 5, 0)], [oracle.agg("count")])[0]
    assert got.tolist() == want.tolist() == [1, 1, 0, 0, 1, 3, 0]


@pytest.mark.parametrize("seed", range(24))
def test_random_host(seed, oracle):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 6000))
    binners, aggs = random_case(rng, n)
    check(binners, aggs, n, oracle)


@pytest.mark.parametrize("seed", range(100, 112))
def test_random_device_resident(seed, oracle):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 6000))
    binners, aggs = random_case(rng, n)
    check(binners, aggs, n, oracle, device=True)


@pytest.mark.parametrize("seed", range(200, 208))
def test_random_chunked(seed, oracle):
    """Chunk boundaries (ragged, unaligned -> scalar-load kernel variant) must not change results."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2000, 9000))
    binners, aggs = random_case(rng, n, allow_first=False)
    want = oracle.binby(binners, aggs, n)
    for chunk, device in ((777, False), (1001, True), (4096, True)):
        got = b200_binby(binners, aggs, n, chunk=chunk, device=device, nthreads=3)
        for a, w, g in zip(aggs, want, got):
            if a["op"] in ("sum", "sum_moment") and np.asarray(a["data"]).dtype.kind == "f":
                assert np.allclose(g, w, rtol=RTOL, atol=1e-9 * max(1.0, float(np.nanmax(np.abs(w)))))
            else:
                assert same(w, g), (a["op"], chunk, device)


def test_first_last_chunked_with_order(oracle):
    """first/last by an order column across chunks: the winner is the smallest (order, global row)."""
    rng = np.random.default_rng(5)
    n = 20000
    x = rng.normal(0, 1, n)
    v = rng.normal(0, 1, n)
    order = rng.integers(0, 50, n).astype("i8")  # many ties -> the row tie-break matters
    binners = [oracle.scalar(x, -3, 3, 16)]
    aggs = [oracle.agg("first", v, None, order=order), oracle.agg("last", v, None, order=order)]
    want = oracle.binby(binners, aggs, n)  # sequential, one chunk
    for chunk in (n, 3000, 1024):
        got = b200_binby(binners, aggs, n, chunk=chunk, device=True, nthreads=3)  # 3 slots = 3 streams: pairs are event-chained
        for w, g in zip(want, got):
            assert same(w, g), chunk


def test_empty_and_tiny(oracle):
    x = np.zeros(0, "f4")
    got = b200_binby([oracle.scalar(x, 0, 1, 4)], [oracle.agg("count"), oracle.agg("min", x)], 0)
    assert got[0].tolist() == [0] * 7
    assert np.all(np.isinf(got[1]))
    x = np.array([0.5], "f4")
    got = b200_binby([oracle.scalar(x, 0, 1, 4)], [oracle.agg("count")], 1)
    assert got[0].tolist() == oracle.binby([oracle.scalar(x, 0, 1, 4)], [oracle.agg("count")], 1)[0].tolist()


def test_bin_edges_bit_exact(oracle):
    """Values sitting on / next to bin edges: the fp64 index math must agree with the reference bit for bit."""
    rng = np.random.default_rng(11)
    bins, vmin, vmax = 1024, -3.0, 3.0
    edges = vmin + (vmax - vmin) * np.arange(bins + 1) / bins
    x64 = np.concatenate([edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf), rng.uniform(-3.1, 3.1, 100000)])
    for dt in ("f8", "f4"):
        x = x64.astype(dt)
        y = rng.permutation(x)
        b = [oracle.scalar(x, vmin, vmax, bins), oracle.scalar(y, vmin, vmax, bins)]
        want = oracle.binby(b, [oracle.agg("count")])[0]
        got = b200_binby(b, [oracle.agg("count")], device=True)[0]
        assert np.array_equal(want, got)
    # awkward limits whose reciprocal is inexact
    x = rng.uniform(0.1, 0.9, 200000)
    b = [oracle.scalar(x, 0.1, 0.9, 7)]
    assert np.array_equal(oracle.binby(b, [oracle.agg("count")])[0], b200_binby(b, [oracle.agg("count")])[0])


def test_headline_shape_sample(oracle):
    """The headline configuration (2-D 1024^2 count on fp32, limits [-3,3]) on a sample the oracle finishes in seconds,
    plus the sum config; large enough (4M rows) to use the global-atomic path and the vectorised loads."""
    rng = np.random.default_rng(42)
    n = 1 << 22
    x, y, z = (rng.normal(0, 1, n).astype("f4") for _ in range(3))
    x[::100003] = np.nan
    b = [oracle.scalar(x, -3, 3, 1024), oracle.scalar(y, -3, 3, 1024)]
    aggs = [oracle.agg("count"), oracle.agg("sum", z), oracle.agg("count", z)]
    want = oracle.binby(b, aggs, n)
    got = b200_binby(b, aggs, n, device=True)
    assert np.array_equal(want[0], got[0])
    assert np.array_equal(want[2], got[2])
    assert np.allclose(got[1], want[1], rtol=RTOL, atol=1e-9)
    assert int(got[0].sum()) == n


def test_tile_partitioned_count_matches_oracle(oracle):
    """count(*) on big grids takes the two-kernel partition path (csrc/ringcount.cu) from 2^22 rows on: check it against the
    oracle for fp32 2-D 1024^2 (32 parts), fp64 3-D 126^3 (64 parts) and a degenerate distribution (one hot cell: the ring of
    its part overflows in every group and the excess rows go to direct REDs)."""
    rng = np.random.default_rng(21)
    n = (1 << 22) + 12345
    x, y = (rng.normal(0, 1, n).astype("f4") for _ in range(2))
    x[::50001] = np.nan
    b = [oracle.scalar(x, -3, 3, 1024), oracle.scalar(y, -3, 3, 1024)]
    assert np.array_equal(oracle.binby(b, [oracle.agg("count")], n)[0], b200_binby(b, [oracle.agg("count")], n, device=True)[0])
    a, c, d = (rng.normal(0, 1, n) for _ in range(3))
    b = [oracle.scalar(a, -3, 3, 126), oracle.scalar(c, -2, 3, 126), oracle.scalar(d, -3, 2, 126)]
    assert np.array_equal(oracle.binby(b, [oracle.agg("count")], n)[0], b200_binby(b, [oracle.agg("count")], n, device=True)[0])
    n = 1 << 23
    x = np.full(n, 0.5, "f4")
    y = np.full(n, -0.25, "f4")
    y[: n // 8] = rng.normal(0, 1, n // 8).astype("f4")
    b = [oracle.scalar(x, -3, 3, 1024), oracle.scalar(y, -3, 3, 1024)]
    got = b200_binby(b, [oracle.agg("count")], n, device=True)[0]
    assert np.array_equal(oracle.binby(b, [oracle.agg("count")], n)[0], got) and int(got.sum()) == n


@pytest.mark.parametrize("case", ["2d_f32_sorted_keys", "1d_f64_64parts", "3d_f32_128parts", "2d_f64_two_hot_parts", "2d_f32_all_nan_y", "2d_f32_ragged"])
def test_ring_partition_variants(case, oracle):
    """csrc/ringcount.cu over its template space (fp32 / fp64 keys, 1-3 dimensions, 32 / 64 parts) and the distributions that
    stress the rings and the chunk lists: keys sorted by the partitioning dimension (every warp fills ONE ring: overflow -> direct
    REDs), two hot parts, a column of NaN (everything in cell row 0), a row count that is no multiple of anything.  The 3-D case's
    grids (160^3 and 153^3 cells) are above the ring's 64 x 49,151 cells: the direct kernel counts them."""
    rng = np.random.default_rng(77)
    n = (1 << 22) + 4097
    if case == "2d_f32_sorted_keys":
        x = rng.normal(0, 1, n).astype("f4")
        y = np.sort(rng.normal(0, 1, n)).astype("f4")
        b = [oracle.scalar(x, -3, 3, 1024), oracle.scalar(y, -3, 3, 1024)]
    elif case == "1d_f64_64parts":
        x = rng.normal(0, 1, n)
        x[::9973] = np.nan
        b = [oracle.scalar(x, -4, 4, 3_000_000)]  # 3,000,003 cells -> 64 parts
    elif case == "3d_f32_128parts":
        x, y, z = (rng.uniform(-1, 1, n).astype("f4") for _ in range(3))
        b = [oracle.scalar(x, -1, 1, 157), oracle.scalar(y, -0.9, 1, 157), oracle.scalar(z, -1, 0.9, 157)]  # 160^3 = 4.096M: >= 2^22 cells, direct path
        got = b200_binby(b, [oracle.agg("count")], n, device=True)[0]
        assert np.array_equal(oracle.binby(b, [oracle.agg("count")], n)[0], got)
        b = [oracle.scalar(x, -1, 1, 150), oracle.scalar(y, -0.9, 1, 150), oracle.scalar(z, -1, 0.9, 150)]  # 153^3 = 3.58M cells -> 128 parts
    elif case == "2d_f64_two_hot_parts":
        x = rng.normal(0, 1, n)
        y = np.where(rng.random(n) < 0.5, 0.001, 2.5) + rng.normal(0, 1e-3, n)
        b = [oracle.scalar(x, -3, 3, 700), oracle.scalar(y, -3, 3, 900)]
    elif case == "2d_f32_all_nan_y":
        x = rng.normal(0, 1, n).astype("f4")
        y = np.full(n, np.nan, "f4")
        y[: n // 16] = rng.normal(0, 1, n // 16).astype("f4")
        b = [oracle.scalar(x, -3, 3, 1024), oracle.scalar(y, -3, 3, 1024)]
    else:
        n = (1 << 23) + 255
        x, y = (rng.standard_t(2, n).astype("f4") for _ in range(2))  # heavy tails: both edge cells busy
        b = [oracle.scalar(x, -3, 3, 2000), oracle.scalar(y, -3, 3, 500)]
    want = oracle.binby(b, [oracle.agg("count")], n)[0]
    got = b200_binby(b, [oracle.agg("count")], n, device=True)[0]
    assert np.array_equal(want, got) and int(got.sum()) == n


def test_grid_larger_than_l2_matches_oracle(oracle):
    """mean+std primitives (count, sum, sum^2) on a grid larger than the L2 at full thresholds (38M rows >= 2^24, 112 MB of
    accumulators): the region-sorted path of csrc/tilesort.cu.  Counts bit-exact, sums within the 1e-6 tolerance."""
    rng = np.random.default_rng(31)
    n = 38_000_000
    x, y, z = (rng.normal(0, 1, n).astype("f4") for _ in range(3))
    v = rng.normal(0, 1, n).astype("f4")
    v[::77777] = np.nan
    b = [oracle.scalar(x, -3, 3, 164), oracle.scalar(y, -3, 3, 164), oracle.scalar(z, -3, 3, 164)]  # 167^3 = 4.66M cells, 3 x 37 MB
    aggs = [oracle.agg("count", v), oracle.agg("sum", v), oracle.agg("sum_moment", v, moment=2)]
    want = oracle.binby(b, aggs, n)
    got = b200_binby(b, aggs, n, device=True)
    assert np.array_equal(want[0], got[0])
    for k in (1, 2):
        assert np.allclose(got[k], want[k], rtol=RTOL, atol=1e-9)


def test_region_sorted_path_matches_oracle(oracle, monkeypatch):
    """grids larger than the L2 take the region-sorted path (csrc/tilesort.cu) from 2^24 rows on; here the thresholds are
    lowered through its environment knobs so that every variant (64 / 128 regions, with and without a value column, fp32 /
    fp64, ragged last tile, NaN keys and values, bucket overflow -> direct application) is checked against the oracle."""
    monkeypatch.setenv("B200_TILESORT_FORCE", "1")
    monkeypatch.setenv("B200_TILESORT_MIN_ROWS", "1000")
    rng = np.random.default_rng(41)
    n = 100_003
    x, y = (rng.normal(0, 1, n).astype("f4") for _ in range(2))
    v = rng.normal(0, 1, n)
    x[::3331] = np.nan
    v[::1777] = np.nan
    b = [oracle.scalar(x, -3, 3, 300), oracle.scalar(y, -3, 3, 300)]
    aggs = [oracle.agg("count", v), oracle.agg("sum", v), oracle.agg("sum_moment", v, moment=2), oracle.agg("count")]
    want = oracle.binby(b, aggs, n)
    for region_kb in (None, "32"):  # default: 45 regions; 32 KB budget: 90 regions (four per lane in the scan)
        if region_kb:
            monkeypatch.setenv("B200_TILESORT_REGION_KB", region_kb)
        for device in (True, False):
            got = b200_binby(b, aggs, n, device=device)
            assert np.array_equal(want[0], got[0]) and np.array_equal(want[3], got[3])
            for k in (1, 2):
                assert np.allclose(got[k], want[k], rtol=RTOL, atol=1e-9)
    monkeypatch.delenv("B200_TILESORT_REGION_KB")
    # no value column, fp64 keys, 3-D
    a, c, d = (rng.normal(0, 1, n) for _ in range(3))
    b = [oracle.scalar(a, -3, 3, 40), oracle.scalar(c, -2, 3, 41), oracle.scalar(d, -3, 2, 42)]
    assert np.array_equal(oracle.binby(b, [oracle.agg("count")], n)[0], b200_binby(b, [oracle.agg("count")], n, device=True)[0])
    # one hot cell: its bucket overflows and the excess is applied directly
    x = np.full(n, 0.5, "f4")
    y = np.full(n, -0.25, "f4")
    vf = rng.normal(0, 1, n).astype("f4")
    b = [oracle.scalar(x, -3, 3, 300), oracle.scalar(y, -3, 3, 300)]
    aggs = [oracle.agg("count", vf), oracle.agg("sum", vf)]
    want, got = oracle.binby(b, aggs, n), b200_binby(b, aggs, n, device=True)
    assert np.array_equal(want[0], got[0]) and int(got[0].sum()) == n
    assert np.allclose(got[1], want[1], rtol=RTOL, atol=1e-9)


def test_large_properties():
    """Full-size style properties that need no oracle: conservation of rows, chunk-sum consistency, idempotent merge."""
    import torch
    from vaex_b200 import superagg
    n = 1 << 26
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(n, device="cuda", dtype=torch.float32, generator=g)
    y = torch.randn(n, device="cuda", dtype=torch.float32, generator=g)

    def count(parts):
        bx = superagg.BinnerScalar_float32(1, "x", -3, 3, 1024)
        by = superagg.BinnerScalar_float32(1, "y", -3, 3, 1024)
        grid = superagg.Grid([bx, by])
        agg = superagg.AggCount_float32(grid, 1, 1)
        for i1, i2 in parts:
            bx.set_data(0, x[i1:i2])
            by.set_data(0, y[i1:i2])
            agg.clear_data_mask(0)
            grid.bin(0, [agg], i2 - i1)
        return agg.get_result()

    whole = count([(0, n)])
    assert int(whole.sum()) == n
    assert whole.shape == (1027, 1027)
    parts = count([(0, n // 3), (n // 3, n // 2 + 1), (n // 2 + 1, n)])  # unaligned split -> scalar-load variant
    assert np.array_equal(whole, parts)
    # cross-check the interior against torch.histogramdd-style binning done in fp64 on the device
    ix = torch.floor((x.double() + 3.0) * (1.0 / 6.0) * 1024).long()
    inside = (x >= -3) & (x < 3)
    assert int(whole[2:-1, :].sum()) == int(inside.sum()) or abs(int(whole[2:-1, :].sum()) - int(inside.sum())) < 4
    del ix


def test_minmax_large_unaligned_masked(oracle):
    """the vectorised limits pre-pass at a size where every code path runs (scalar head, 4-deep vector body, tail; masks; a view
    that starts off a 16-byte boundary), all dtypes, against the oracle"""
    from helpers import to_device
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(5)
    n = (1 << 22) + 77
    for dt in ("f8", "f4", "i8", "i4", "i2", "i1", "u1", "?"):
        d = np.dtype(dt)
        if d.kind == "f":
            v = rng.standard_normal(n).astype(d)
            v[::997] = np.nan
        elif d.kind == "b":
            v = rng.integers(0, 2, n).astype(d)
        else:
            info = np.iinfo(d)
            v = rng.integers(info.min, info.max, n, dtype=np.int64, endpoint=True).astype(d)
        for off in (0, 3):
            w = v[off:]
            want = oracle.minmax(w, raw=True)
            assert np.array_equal(Frame({"v": w}).minmax("v", raw=True), want, equal_nan=True), (dt, off, "host")
            assert np.array_equal(Frame({"v": to_device(v)[off:]}).minmax("v", raw=True), want, equal_nan=True), (dt, off, "device")
        m = rng.random(n) < 0.5
        assert np.array_equal(Frame({"v": np.ma.array(v, mask=m)}).minmax("v", raw=True), oracle.minmax(np.ma.array(v, mask=m), raw=True), equal_nan=True)


def test_bin_index_sweep_all_fp32(oracle):
    """EVERY one of the 2^32 float32 bit patterns (both zeros, denormals, +-inf, every NaN payload) through the ONE device
    ``bin_index`` (csrc/device_utils.cuh) and through the clamped magic-floor variant the ring partition uses for float32 keys
    (csrc/ringcount.cu), against the oracle's restatement of BinnerScalar::to_bins (src/binners.cpp:13-57).  x walks the patterns
    in order, y walks them through an odd-multiplier bijection, so both dimensions (different vmin / vmax / bins) see all of
    them; the 2-D grid goes down the ring path (2^28 rows a call), its x marginal down the small-grid kernel of csrc/fast.cu."""
    from concurrent.futures import ThreadPoolExecutor
    step = 1 << 28

    def chunk(k):
        i = np.arange(k * step, (k + 1) * step, dtype=np.uint64)
        x = i.astype(np.uint32).view(np.float32)
        y = ((i * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32)
        return x, y

    def want(k):
        x, y = chunk(k)
        return oracle.binby([oracle.scalar(x, -3.25, 7.5, 1500), oracle.scalar(y, -1e-3, 2.5e-3, 700)], [oracle.agg("count")], step)[0]

    total = np.int64(0)
    with ThreadPoolExecutor(8) as pool:  # the oracle is C behind ctypes: the GIL is released
        futures = [pool.submit(want, k) for k in range(16)]
        for k in range(16):
            x, y = chunk(k)
            got = b200_binby([oracle.scalar(x, -3.25, 7.5, 1500), oracle.scalar(y, -1e-3, 2.5e-3, 700)], [oracle.agg("count")], step, device=True)[0]
            got_x = b200_binby([oracle.scalar(x, -3.25, 7.5, 1500)], [oracle.agg("count")], step, device=True)[0]
            w = futures[k].result()
            assert np.array_equal(w, got), f"patterns {k * step:#x}..{(k + 1) * step:#x}"
            axis = 1 if w.shape[0] == got_x.shape[0] else 0
            assert np.array_equal(w.sum(axis=axis), got_x)
            total += got.sum()
    assert int(total) == 1 << 32


def test_ring_partition_more_than_one_batch_is_linear():
    """More than 2^30 rows in ONE call: csrc/ringcount.cu cuts the call into equal batches (32-bit entry counts).  Size-independent
    property instead of a 9 GB host oracle pass: the grid of the whole call equals the sum of the grids of two calls that each fit
    one batch, and the grid's total equals the row count."""
    import torch
    from vaex_b200 import superagg
    n = (1 << 30) + 77_777
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    y = torch.empty(n, dtype=torch.float32, device="cuda").normal_(generator=gen)
    bx = superagg.BinnerScalar_float32(1, "x", -3, 3, 1024)
    by = superagg.BinnerScalar_float32(1, "y", -3, 3, 1024)
    grid = superagg.Grid([bx, by])

    def count(lo, hi):
        agg = superagg.AggCount_int64(grid, 1, 1)
        bx.set_data(0, x[lo:hi])
        by.set_data(0, y[lo:hi])
        grid.bin(0, [agg], hi - lo)
        return agg.get_result()
    whole = count(0, n)
    cut = 600_000_003
    parts = count(0, cut) + count(cut, n)
    assert int(whole.sum()) == n and np.array_equal(whole, parts)
