"""Every per-slot call that takes a memspace gives the same result whichever way its inputs are placed: pageable host (HOST),
device (DEVICE), page-locked host next to device columns (MIXED) and page-locked host (HOST).  A MIXED call without
B200_FLAG_ASYNC_HOST returns only once its stream is idle, so the caller may overwrite its host buffers right away.  The calls
that take a device grid (percentile, mutual information) give the same result in host and in device memory.  Every entry point
rejects an out-of-range slot naming the call, and nothing stays allocated."""
import ctypes as C
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 200_003
WAYS = ("host", "device", "mixed", "pinned")


def _data():
    rng = np.random.default_rng(7)
    words = np.array(["k%d" % k for k in rng.integers(0, 3000, 50_000)])
    return dict(
        keys=rng.integers(0, 1000, N).astype(np.int64),
        keys2=rng.integers(0, 50, N).astype(np.int64),
        vals=rng.integers(-1000, 1000, N).astype(np.float64),  # integral: every sum is exact whatever the order of the atomics
        vals2=rng.integers(-1000, 1000, N).astype(np.float64),
        x=rng.random(N),
        mask=(rng.random(N) < 0.1).astype(np.uint8),
        offsets=np.concatenate([[0], np.cumsum([len(w) for w in words])]).astype(np.int64),
        bytes=np.frombuffer("".join(words).encode(), np.uint8).copy(),
        smask=(rng.random(len(words)) < 0.05).astype(np.uint8),
    )


class Placed:
    """The columns of one call placed for one way; in `mixed` the first column is page-locked host memory, the others device."""

    def __init__(self, way, *arrays):
        import torch
        from vaex_b200 import _lib
        self.way, self.cols, self.host, self.pins = way, [], [], []
        for i, a in enumerate(arrays):
            if way == "device" or (way == "mixed" and i > 0):
                self.cols.append(torch.from_numpy(np.ascontiguousarray(a)).cuda())
                continue
            h = np.array(a, copy=True)
            if way != "host":
                self.pins.append(_lib.pinned(h))
                self.host.append(h)
            self.cols.append(h)
        torch.cuda.synchronize()
        self.memspace = {"host": _lib.MEM_HOST, "device": _lib.MEM_DEVICE, "mixed": _lib.MEM_MIXED, "pinned": _lib.MEM_HOST}[way]

    def __getitem__(self, i):
        c = self.cols[i]
        return c.data_ptr() if hasattr(c, "data_ptr") else c.ctypes.data

    def returned(self, ctx):
        """after the call: a MIXED call has nothing left on its stream, and overwriting its host columns changes nothing"""
        import torch
        if self.way == "mixed":
            assert torch.cuda.ExternalStream(ctx.stream(0)).query(), "a MIXED call returned while its stream was busy"
            for h in self.host:
                h.view(np.uint8)[:] = 0xA5

    def release(self, ctx):
        ctx.sync()
        for p in self.pins:
            p.release()


def _out(way, n, dtype, device):
    import torch
    if device:
        return torch.zeros(max(n, 1) * np.dtype(dtype).itemsize, dtype=torch.uint8, device="cuda")
    return np.zeros(max(n, 1), dtype)


def _ptr(o):
    return o.data_ptr() if hasattr(o, "data_ptr") else o.ctypes.data


def _host(o, n, dtype):
    return o.cpu().numpy().view(dtype)[:n].copy() if hasattr(o, "data_ptr") else o[:n].copy()


def _set(ctx, keys):
    from vaex_b200 import _lib
    h = C.c_void_p()
    _lib.check(_lib.lib().b200_set_create(ctx._h, _lib.I64, 1, -1, C.byref(h)))
    _lib.check(_lib.lib().b200_set_update(h, 0, keys.ctypes.data, None, len(keys), 0, 0, None, None, _lib.MEM_HOST, 0))
    return h


def _strset(ctx, d, n):
    from vaex_b200 import _lib
    h = C.c_void_p()
    _lib.check(_lib.lib().b200_strset_create(ctx._h, 1, -1, C.byref(h)))
    off = d["offsets"][:n + 1]
    _lib.check(_lib.lib().b200_strset_update(h, 0, off.ctypes.data, d["bytes"].ctypes.data, None, n, 0, None, None, _lib.MEM_HOST))
    return h


def run_bin(ctx, d, way):
    from vaex_b200 import _lib
    L = _lib.lib()
    p = Placed(way, d["keys"], d["vals"], d["mask"])
    cells = 1000 + 2
    aggs = []
    for op in (_lib.AGG_COUNT, _lib.AGG_SUM):
        h = C.c_void_p()
        _lib.check(L.b200_agg_create(ctx._h, op, _lib.F64, _lib.F64, 0, 0, cells, C.byref(h)))
        aggs.append(h)
    B = (_lib.Binner * 1)()
    B[0].kind, B[0].dtype, B[0].ordinal_count, B[0].min_value, B[0].data = _lib.BINNER_ORDINAL, _lib.I64, 1000, 0, p[0]
    A = (_lib.AggInput * 2)()
    for k, h in enumerate(aggs):
        A[k].agg, A[k].data, A[k].mask = h, p[1], p[2]
    _lib.check(L.b200_bin(ctx._h, 0, B, 1, A, 2, N, 0, p.memspace, 0))
    p.returned(ctx)
    count, total = np.empty(cells, np.int64), np.empty(cells, np.float64)
    _lib.check(L.b200_agg_read(aggs[0], count.ctypes.data, None))
    _lib.check(L.b200_agg_read(aggs[1], total.ctypes.data, None))
    for h in aggs:
        L.b200_agg_destroy(h)
    p.release(ctx)
    return count, total


def run_eval(ctx, d, way):
    from vaex_b200 import _lib
    p = Placed(way, d["vals"], d["vals2"])
    prog = (_lib.ExprOp * 3)()
    prog[0].op, prog[0].arg = 0, 0  # B200_EX_INPUT 0
    prog[1].op, prog[1].arg = 0, 1  # B200_EX_INPUT 1
    prog[2].op = 3  # B200_EX_ADD in float64
    inputs = (_lib.ExprInput * 2)()
    for k in range(2):
        inputs[k].data, inputs[k].dtype = p[k], _lib.F64
    out = _out(way, N, np.float64, True)
    _lib.check(_lib.lib().b200_eval(ctx._h, 0, prog, 3, inputs, 2, None, 0, N, p.memspace, _lib.F64, out.data_ptr()))
    p.returned(ctx)
    ctx.sync()
    p.release(ctx)
    return _host(out, N, np.float64)


def run_compact(ctx, d, way):
    from vaex_b200 import _lib
    p = Placed(way, d["mask"], d["vals"])
    out = _out(way, N, np.float64, True)
    count = C.c_int64(-1)
    _lib.check(_lib.lib().b200_compact(ctx._h, 0, p[0], 1, (C.c_void_p * 1)(p[1]), (C.c_int32 * 1)(_lib.F64), N, p.memspace,
                                       (C.c_void_p * 1)(out.data_ptr()), C.byref(count)))
    p.returned(ctx)
    ctx.sync()
    p.release(ctx)
    return count.value, _host(out, count.value, np.float64)


def run_minmax(ctx, d, way):
    from vaex_b200 import _lib
    p = Placed(way, d["vals"], d["mask"])
    out = np.empty(2, np.float64)
    _lib.check(_lib.lib().b200_minmax(ctx._h, 0, _lib.F64, 0, p[0], p[1], N, p.memspace, out.ctypes.data))
    p.returned(ctx)
    p.release(ctx)
    return out


def run_stat(ctx, d, way):
    from vaex_b200 import _lib, statistic
    p = Placed(way, d["x"], d["vals"])
    st = statistic.Statistic(4, _lib.F64, [8], [0.0], [1.0], False, 1, 1, ctx=ctx)  # B200_STAT_MOMENTS_012
    st.bin(0, [p.cols[0]], [p.cols[1]], [None], N, 0)
    p.returned(ctx)
    out = st.read()
    st.close()
    p.release(ctx)
    return out


def run_set_update(ctx, d, way):
    from vaex_b200 import _lib
    L = _lib.lib()
    p = Placed(way, d["keys"], d["mask"])
    h = C.c_void_p()
    _lib.check(L.b200_set_create(ctx._h, _lib.I64, 1, -1, C.byref(h)))
    _lib.check(L.b200_set_update(h, 0, p[0], p[1], N, 0, 0, None, None, p.memspace, 0))
    p.returned(ctx)
    keys = np.empty(L.b200_set_count(h), np.int64)
    _lib.check(L.b200_set_key_array(h, keys.ctypes.data))
    L.b200_set_destroy(h)
    p.release(ctx)
    return keys


def run_set_map(ctx, d, way, isin):
    from vaex_b200 import _lib
    L = _lib.lib()
    h = _set(ctx, d["keys"][:N // 2])
    dt = np.uint8 if isin else {_lib.I8: np.int8, _lib.I16: np.int16, _lib.I32: np.int32, _lib.I64: np.int64}[L.b200_set_ordinal_dtype(h)]
    p = Placed(way, d["keys"])
    out = _out(way, N, dt, way != "host")  # page-locked keys with a device result: a HOST call writing to the device
    fn = L.b200_set_isin if isin else L.b200_set_map_ordinal
    _lib.check(fn(h, 0, p[0], N, _ptr(out), p.memspace, 0))
    p.returned(ctx)
    ctx.sync()
    L.b200_set_destroy(h)
    p.release(ctx)
    return _host(out, N, dt)


def run_combine(ctx, d, way):
    from vaex_b200 import _lib
    L = _lib.lib()
    sets = [_set(ctx, d["keys"][:N // 2]), _set(ctx, d["keys2"][:N // 2])]
    p = Placed(way, d["keys"], d["keys2"], d["mask"])
    out = _out(way, N, np.int64, way != "host")
    _lib.check(L.b200_set_combine(ctx._h, 0, 2, (C.c_void_p * 2)(*[s.value for s in sets]), (C.c_void_p * 2)(p[0], p[1]),
                                  (C.c_void_p * 2)(p[2], None), (C.c_int64 * 2)(1, 1003), N, _ptr(out), p.memspace, 0))
    p.returned(ctx)
    ctx.sync()
    for s in sets:
        L.b200_set_destroy(s)
    p.release(ctx)
    return _host(out, N, np.int64)


def run_strset_update(ctx, d, way):
    from vaex_b200 import _lib
    L = _lib.lib()
    n = len(d["smask"])
    p = Placed(way, d["offsets"], d["bytes"], d["smask"])
    h = C.c_void_p()
    _lib.check(L.b200_strset_create(ctx._h, 1, -1, C.byref(h)))
    vals, mi = np.empty(n, np.int64), np.empty(n, np.int16)
    _lib.check(L.b200_strset_update(h, 0, p[0], p[1], p[2], n, 1, vals.ctypes.data, mi.ctypes.data, p.memspace))
    p.returned(ctx)
    L.b200_set_destroy(h)
    p.release(ctx)
    return vals, mi


def run_strset_map(ctx, d, way):
    from vaex_b200 import _lib
    L = _lib.lib()
    n = len(d["smask"])
    h = _strset(ctx, d, n // 2)
    p = Placed(way, d["offsets"], d["bytes"], d["smask"])
    out = _out(way, n, np.int64, way != "host")
    _lib.check(L.b200_strset_map_ordinal(h, 0, p[0], p[1], p[2], n, _ptr(out), p.memspace, int(way != "host")))
    p.returned(ctx)
    ctx.sync()
    L.b200_set_destroy(h)
    p.release(ctx)
    return _host(out, n, np.int64)


RUNS = dict(bin=run_bin, eval=run_eval, compact=run_compact, minmax=run_minmax, stat_bin=run_stat, set_update=run_set_update,
            set_map_ordinal=lambda c, d, w: run_set_map(c, d, w, False), set_isin=lambda c, d, w: run_set_map(c, d, w, True),
            set_combine=run_combine, strset_update=run_strset_update, strset_map_ordinal=run_strset_map)


def _live(ctx):
    gc.collect()
    ctx.sync()
    return ctx.mem_stats()["live"]


def _same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=np.asarray(a).dtype.kind == "f")


@pytest.mark.parametrize("call", sorted(RUNS))
def test_every_placement_gives_the_same_result(call):
    from vaex_b200 import _lib
    ctx = _lib.context()
    d = _data()
    base = _live(ctx)
    results = {way: RUNS[call](ctx, d, way) for way in WAYS}
    for way in WAYS[1:]:
        assert _same(results[way], results["host"]), (call, way)
    assert _live(ctx) == base


def test_grid_finishes_in_host_and_device_memory():
    import torch
    from vaex_b200 import _lib, mutual_information, percentile
    ctx = _lib.context()
    base = _live(ctx)
    rng = np.random.default_rng(3)
    grid = torch.from_numpy(rng.integers(0, 50, (40, 11)).astype(np.int64)).cuda()  # binby (first, fastest) x percentile axis
    host = percentile.grid_percentile(grid.data_ptr(), [11, 40], 0.0, 1.0, [10.0, 50.0, 90.0])
    dev = torch.zeros(host.size, dtype=torch.float64, device="cuda")
    percentile.grid_percentile(grid.data_ptr(), [11, 40], 0.0, 1.0, [10.0, 50.0, 90.0], out=dev)
    assert np.array_equal(dev.cpu().numpy(), host.ravel())
    for sizes in ([7, 7, 260], [7, 7, 5]):  # one CTA per cell, and the split regime
        g = torch.from_numpy(rng.integers(0, 20, int(np.prod(sizes))).astype(np.int64)).cuda()
        host = mutual_information.grid_mutual_information(g.data_ptr(), sizes, 2)
        dev = torch.zeros(host.size, dtype=torch.float64, device="cuda")
        mutual_information.grid_mutual_information(g.data_ptr(), sizes, 2, out=dev)
        assert np.array_equal(dev.cpu().numpy(), host)
    del grid, g
    assert _live(ctx) == base


def test_out_of_range_slot_names_the_call():
    import torch
    from vaex_b200 import _lib, statistic
    L = _lib.lib()
    ctx = _lib.context()
    H = _lib.MEM_HOST
    s = _set(ctx, np.arange(10, dtype=np.int64))
    ss = _strset(ctx, _data(), 10)
    st = statistic.Statistic(1, _lib.F64, [8], [0.0], [1.0], False, 1, 1, ctx=ctx)
    col = (statistic.StatColumn * 1)()
    col[0].dtype = _lib.F64
    grid = torch.zeros(64, dtype=torch.int64, device="cuda")
    out = np.zeros(64, np.float64)
    count = C.c_int64()
    prog = (_lib.ExprOp * 1)()
    prog[0].op = 1  # B200_EX_CONST_F64
    calls = {
        "b200_bin": lambda k: L.b200_bin(ctx._h, k, None, 0, None, 0, 0, 0, H, 0),
        "b200_eval": lambda k: L.b200_eval(ctx._h, k, prog, 1, None, 0, None, 0, 0, H, _lib.F64, None),
        "b200_compact": lambda k: L.b200_compact(ctx._h, k, None, 0, None, None, 0, H, None, C.byref(count)),
        "b200_minmax": lambda k: L.b200_minmax(ctx._h, k, _lib.F64, 0, None, None, 0, H, out.ctypes.data),
        "b200_stat_bin": lambda k: L.b200_stat_bin(st._h, k, col, col, None, 0, 0, H, 0),
        "b200_set_update": lambda k: L.b200_set_update(s, k, None, None, 0, 0, 0, None, None, H, 0),
        "b200_set_map_ordinal": lambda k: L.b200_set_map_ordinal(s, k, None, 0, None, H, 0),
        "b200_set_isin": lambda k: L.b200_set_isin(s, k, None, 0, None, H, 0),
        "b200_set_combine": lambda k: L.b200_set_combine(ctx._h, k, 1, (C.c_void_p * 1)(s.value), (C.c_void_p * 1)(None), None,
                                                         (C.c_int64 * 1)(1), 0, None, H, 0),
        "b200_strset_update": lambda k: L.b200_strset_update(ss, k, None, None, None, 0, 0, None, None, H),
        "b200_strset_map_ordinal": lambda k: L.b200_strset_map_ordinal(ss, k, None, None, None, 0, None, H, 0),
        "b200_grid_percentile": lambda k: L.b200_grid_percentile(ctx._h, k, grid.data_ptr(), 2, (C.c_int64 * 2)(4, 16), 0.0, 1.0,
                                                                 (C.c_double * 1)(50.0), (C.c_uint8 * 1)(0), 1, H, out.ctypes.data),
        "b200_grid_mutual_information": lambda k: L.b200_grid_mutual_information(ctx._h, k, grid.data_ptr(), 3, (C.c_int64 * 3)(4, 4, 4), 2, H,
                                                                                 out.ctypes.data),
    }
    for name, call in calls.items():
        for k in (ctx.nslots, -1):
            with pytest.raises(RuntimeError, match=name + ": invalid slot"):
                _lib.check(call(k))
        _lib.check(call(0))  # the same call on a valid slot does nothing and succeeds
    st.close()
    L.b200_set_destroy(s)
    L.b200_set_destroy(ss)
