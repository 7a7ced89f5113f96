"""Every device block an operation takes from the context's cache is given back: after each family of operations has run and its
objects were destroyed, the bytes handed out (b200_ctx_mem_stats) are where they started, and repeating the sequence neither leaks
nor grows the cache.  Requests larger than the device are refused with MemoryError and leave the context usable."""
import ctypes as C
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _aggregators(rng):
    import pyarrow as pa
    from vaex_b200 import superagg
    n = 50_000
    x = rng.integers(0, 10, n).astype(np.int32)
    v = rng.normal(size=n)
    b = superagg.BinnerOrdinal_int32(1, "x", 10, 0, False, False)
    g = superagg.Grid([b])
    b.set_data(0, x)
    aggs = [superagg.AggCount_float64(g, 1, 1), superagg.AggSum_float64(g, 1, 1), superagg.AggSumMoment_float64(g, 1, 1, 2),
            superagg.AggMin_float64(g, 1, 1), superagg.AggMax_float64(g, 1, 1), superagg.AggFirst_float64_int64(g, 1, 1, False),
            superagg.AggFirst_float64_int64(g, 1, 1, True)]
    order = np.arange(n, dtype=np.int64)
    for a in aggs:
        a.set_data(0, v)
        if "First" in type(a).__name__:
            a.set_data(0, order, 1)
    g.bin(0, aggs, n)
    for a in aggs:
        a.get_result()
    # merge on one device, FIRST/LAST included
    others = [superagg.AggSum_float64(g, 1, 1), superagg.AggFirst_float64_int64(g, 1, 1, False)]
    for a in others:
        a.set_data(0, v)
    others[1].set_data(0, order, 1)
    g.bin(0, others, n)
    aggs[1].merge([others[0]])
    aggs[5].merge([others[1]])
    # nunique through a table growth: the second call's new pairs no longer fit the table sized for the first
    nu = superagg.AggNUnique_int64(g, 1, 1, False, False)
    for _ in range(2):
        big = rng.integers(0, 1 << 40, 200_000).astype(np.int64)
        b.set_data(0, rng.integers(0, 10, len(big)).astype(np.int32))
        nu.set_data(0, big)
        g.bin(0, [nu], len(big))
    assert nu.get_result().sum() > 350_000
    # numeric and string lists, the string one long enough that the offsets' scan recurses (> 2048 elements)
    b.set_data(0, x)
    lst = superagg.AggList_float64_int64(g, 1, 1)
    lst.set_data(0, v)
    g.bin(0, [lst], n)
    lst.get_result()
    words = pa.array(["w%d" % i for i in rng.integers(0, 1000, n)], type=pa.large_string())
    sl = superagg.AggList_string_int64(g, 1, 1)
    sl.set_data(0, words)
    g.bin(0, [sl], n)
    assert sum(len(c) for c in sl.get_result().to_pylist()) == n


def _sets(rng):
    from vaex_b200 import _lib, superutils
    keys = rng.integers(0, 5000, 100_000).astype(np.int64)
    s = superutils.ordered_set_int64(3)
    s.update(keys, -1, return_values=True)
    s.map_ordinal(keys)
    s.isin(keys)
    s.key_array()
    c = superutils.counter_int64(2)
    c.update(keys)
    c.counts()
    c2 = superutils.counter_int64(2)
    c2.update(keys[:100] + 7000)
    c.merge([c2])
    c.counts()
    fk = superutils.ordered_set_int64(np.arange(100, dtype=np.int64), -1, 0, 0, "")
    t = superutils.ordered_set_int64(3)
    t.update(keys[:1000] + 10_000)
    s.merge([t])
    s.key_array()
    # combine into host memory
    ctx = _lib.context()
    out = np.empty(len(keys), np.int64)
    sets = (C.c_void_p * 1)(s._h.value)
    cols = (C.c_void_p * 1)(keys.ctypes.data)
    _lib.check(_lib.lib().b200_set_combine(ctx._h, 0, 1, sets, cols, None, (C.c_int64 * 1)(1), len(keys), out.ctypes.data, _lib.MEM_HOST, 0))
    strs = np.array(["k%d" % i for i in keys[:20_000]], dtype=object)
    ss = superutils.ordered_set_string(2)
    ss.update(strs, return_values=True)
    ss.map_ordinal(strs)
    ss.key_array()
    del s, c, c2, fk, t, ss


def _finishes(rng):
    import torch
    from vaex_b200 import _lib, expression, mutual_information, percentile, statistic
    keep = (rng.random(100_000) < 0.3).astype(np.uint8)
    count, _ = expression.compact(0, keep, [rng.normal(size=100_000)])
    assert count == int(keep.sum())
    st = statistic.Statistic(1, _lib.F64, [8], [0.0], [1.0], False, 1, 1)  # B200_STAT_COUNT of one weight
    x = rng.random(10_000)
    st.bin(0, [x], [x], [None], len(x), 0)
    st.read()
    st.close()
    grid = torch.from_numpy(rng.integers(0, 50, (8, 5)).astype(np.int64)).cuda()  # binby (first, fastest) x percentile axis
    percentile.grid_percentile(grid.data_ptr(), [5, 8], 0.0, 1.0, [10.0, 50.0, 90.0])
    # mutual information in both regimes: one CTA per cell (>= 256 binby cells) and the split regime (2 binby cells)
    for sizes in ([7, 7, 260], [7, 7, 5]):
        g = torch.from_numpy(rng.integers(0, 20, int(np.prod(sizes))).astype(np.int64)).cuda()
        mutual_information.grid_mutual_information(g.data_ptr(), sizes, 2)
    torch.cuda.synchronize()


def _live(ctx):
    gc.collect()
    ctx.sync()
    return ctx.mem_stats()


def test_every_block_is_given_back():
    from vaex_b200 import _lib
    ctx = _lib.context()
    base = _live(ctx)["live"]
    cached = []
    for _ in range(3):
        rng = np.random.default_rng(1)  # the same sizes every round: a second round finds every block it needs in the cache
        for step in (_aggregators, _sets, _finishes):
            step(rng)
            assert _live(ctx)["live"] == base, step.__name__
        cached.append(_live(ctx)["cached"])
    assert cached[2] <= cached[0] and cached[1] <= cached[0], cached


def test_out_of_memory_is_memory_error():
    import torch
    from vaex_b200 import _lib
    ctx = _lib.context()
    total = torch.cuda.get_device_properties(ctx.device).total_memory
    before = _live(ctx)["live"]
    cells = total // 8 * 2  # int64 counts: twice the device
    h = C.c_void_p()
    with pytest.raises(MemoryError, match=str(cells * 8)):
        _lib.check(_lib.lib().b200_agg_create(ctx._h, _lib.AGG_COUNT, _lib.F64, _lib.I64, 0, 0, cells, C.byref(h)))
    assert _live(ctx)["live"] == before
    sizes = (C.c_int64 * 2)(1 << 30, 64)  # 2^36 cells of one count: 512 GB
    lo, hi = (C.c_double * 2)(0, 0), (C.c_double * 2)(1, 1)
    with pytest.raises(MemoryError, match=str((1 << 36) * 8)):
        _lib.check(_lib.lib().b200_stat_create(ctx._h, 0, _lib.F64, 2, sizes, lo, hi, 0, 0, 1, C.byref(h)))
    assert _live(ctx)["live"] == before
    _aggregators(np.random.default_rng(2))  # the context still works
    assert _live(ctx)["live"] == before
