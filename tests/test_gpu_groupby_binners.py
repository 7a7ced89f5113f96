"""Frame.groupby with Binner, BinnerInteger and BinnerTime on the device, against numpy and the time binner's numpy restatement
(time_binner_oracle.py)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]
import groupby_binner_cases as GC  # noqa: E402
import time_binner_oracle as TB  # noqa: E402

pytestmark = pytest.mark.gpu


class DeviceDatetime:
    """a datetime64 column in device memory: a torch int64 tensor exposed with the datetime typestr"""

    def __init__(self, tensor, dtype):
        self.t, self.dtype = tensor, np.dtype(dtype)
        self.__cuda_array_interface__ = dict(tensor.__cuda_array_interface__, typestr=self.dtype.str)

    def __len__(self):
        return len(self.t)

    def __getitem__(self, s):
        return DeviceDatetime(self.t[s], self.dtype)


def place(columns, where):
    """columns on the host, page-locked, or (plain numeric and datetime ones) on the device"""
    import pyarrow as pa
    import torch
    columns = {k: pa.array(v.tolist(), type=pa.large_string()) if isinstance(v, np.ndarray) and v.dtype.kind == "O" else v for k, v in columns.items()}
    if where != "device":
        return columns
    out = {}
    for k, v in columns.items():
        if isinstance(v, np.ndarray) and not np.ma.isMaskedArray(v) and v.dtype.kind in "biufM" and v.dtype.isnative:
            t = torch.from_numpy(np.ascontiguousarray(v.view(np.int64) if v.dtype.kind == "M" else v)).cuda()
            out[k] = DeviceDatetime(t, v.dtype) if v.dtype.kind == "M" else t
        else:
            out[k] = v
    return out


def frame(columns, where="host", filter=None):
    from vaex_b200.frame import Frame
    return Frame(place(columns, where), pin=where == "pinned", filter=filter)


def host(a):
    if hasattr(a, "__cuda_array_interface__") and not isinstance(a, np.ndarray):
        import torch
        return torch.as_tensor(a, device="cuda").cpu().numpy()
    return a


def reference_limits(t, keep):
    """the reference's (tmin, tmax): float32 statistic of the signed ticks of the kept non-NaT rows, cast back (truncation)"""
    v = t[keep & ~np.isnat(t)]
    f = v.astype(np.int64).astype(np.float32).astype(np.float64)
    return np.array([f.min(), f.max()]).astype(t.dtype)


def expected_time(t, res, every, keep=None, masked=None):
    """(keys, cell of every row or -1) of BinnerTime over the rows `keep`"""
    keep = np.ones(len(t), bool) if keep is None else keep
    masked = np.zeros(len(t), bool) if masked is None else masked
    unit = np.datetime_data(t.dtype)[0]
    tmin, tmax = reference_limits(t, keep & ~masked)
    begin, end = (int(x.astype(f"M8[{res}]").astype(np.int64)) for x in (tmin, tmax))
    n = (end - begin + every) // every
    cells = TB.bins(t.astype(np.int64), unit, res, begin, every, n, masked)
    cells = np.where(keep & (cells < n), cells, -1)
    return np.arange(np.datetime64(begin, res), np.datetime64(end, res) + 1, every), cells


def grouped(cells, values, fn):
    """per cell with rows, in cell order: fn(values of the cell)"""
    used = np.unique(cells[cells >= 0])
    return used, [fn(values[cells == c]) for c in used]


def make_binner(df, key):
    from vaex_b200.frame import Binner, BinnerInteger, BinnerTime
    if isinstance(key, str):
        return key
    if key[0] == "time":
        return BinnerTime(key[1], key[2], df=df, every=key[3])
    if key[0] == "binner":
        return Binner(key[1], key[2], key[3], key[4], df=df)
    return BinnerInteger(key[1], df=df, **key[2])


def tolist(a):
    return a.tolist() if hasattr(a, "tolist") else list(a)


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("case", GC.CASES, ids=[c[0] for c in GC.CASES])
def test_reference_case(case, where):
    from vaex_b200 import agg as A
    name, columns, keys, agg, expected, kwargs = case
    df = frame(columns, where)
    by = [make_binner(df, k) for k in keys]
    a = {"count": "count", "sum": {"sum": A.sum(agg[-1])}, "nunique": {"c": A.nunique(agg[-1])}, "list": {"l": A.list(agg[-1])}}[agg[0]]
    if name == "datetime_per_week":
        a = {"y": "sum"}
    out = df.groupby(by if len(by) > 1 else by[0], agg=a, **kwargs)
    if "__len__" in expected:
        assert len(out["sum"]) == expected["__len__"] and int(np.sum(out["sum"])) == expected["__sum__"]
        return
    value = [k for k in expected if not k.startswith("__")][-1]
    for k, want in expected.items():
        if k.startswith("__"):
            continue
        got = out[{"y": "y_sum", "c": "c", "sum": "sum", "count": "count"}.get(k, k) if k == value else k]
        assert tolist(got) == (pytest.approx(want) if isinstance(want[0], float) else want), k
    if "__first_list__" in expected:
        assert set(out["l"][0].as_py()) == expected["__first_list__"]


def datetimes(rng, n, unit="ns", lo="1950-01-01", hi="2030-01-01"):
    a, b = (int(np.datetime64(x).astype(f"M8[{unit}]").astype(np.int64)) for x in (lo, hi))
    return rng.integers(a, b, n).astype(f"M8[{unit}]")


@pytest.mark.parametrize("where", ["host", "device", "pinned", "big-endian"])
def test_every_aggregator_through_a_time_key(where):
    from vaex_b200 import agg as A
    from vaex_b200.frame import BinnerTime
    rng = np.random.default_rng(1)
    n = 20_000
    t = datetimes(rng, n)
    y = rng.standard_normal(n)
    k = rng.integers(0, 50, n)
    o = rng.permutation(n)  # a distinct order per row: first / last are the rows of the smallest / largest order
    s = np.array([f"s{v}" for v in rng.integers(0, 9, n)], dtype=object)
    cols = {"t": t.astype(">M8[ns]") if where == "big-endian" else t, "y": y, "k": k, "o": o, "s": s}
    df = frame(cols, "host" if where == "big-endian" else where)
    try:
        check_every_aggregator(df, t, y, k, o, s)
    finally:
        if df._pinned is not None:
            df._pinned.release()  # unregister before the arrays are freed


def check_every_aggregator(df, t, y, k, o, s):
    from vaex_b200 import agg as A
    from vaex_b200.frame import BinnerTime
    out = df.groupby(BinnerTime.per_month("t", df=df), agg={"c": A.count(), "sum": A.sum("y"), "mean": A.mean("y"), "std": A.std("y"),
                                                           "min": A.min("y"), "max": A.max("y"), "first": A.first("y", "o"), "last": A.last("y", "o"),
                                                           "nu": A.nunique("k"), "l": A.list("k"), "ls": A.list("s")})
    keys, cells = expected_time(t, "M", 1)
    used, counts = grouped(cells, y, len)
    np.testing.assert_array_equal(out["t"], keys[used])
    assert out["t"].dtype == np.dtype("M8[M]")
    np.testing.assert_array_equal(out["c"], counts)
    np.testing.assert_allclose(out["sum"], grouped(cells, y, np.sum)[1], rtol=1e-10)
    np.testing.assert_allclose(out["mean"], grouped(cells, y, np.mean)[1], rtol=1e-10)
    np.testing.assert_allclose(out["std"], grouped(cells, y, np.std)[1], rtol=1e-8)
    np.testing.assert_array_equal(out["min"], grouped(cells, y, np.min)[1])
    np.testing.assert_array_equal(out["max"], grouped(cells, y, np.max)[1])
    np.testing.assert_array_equal(out["nu"], grouped(cells, k, lambda v: len(np.unique(v)))[1])
    for c, f, l_, ls in zip(used, np.asarray(out["first"]), np.asarray(out["last"]), range(len(used))):
        rows = np.nonzero(cells == c)[0]
        assert f == y[rows[np.argmin(o[rows])]]
        assert l_ == y[rows[np.argmax(o[rows])]]
        assert sorted(out["l"][ls].as_py()) == sorted(k[rows].tolist())
        assert sorted(out["ls"][ls].as_py()) == sorted(s[rows].tolist())


# per resolution, the span of the data: wide for the calendar units, a window around 1970-01-01 (pre-1970 rows included) for the
# fine ones, so that every grid stays small
SPANS = {"Y": None, "M": None, "W": None, "D": None, "h": ("1995-01-01", "2005-01-01"), "m": 3 * 86400 * 10 ** 9, "s": 86400 * 10 ** 9,
         "ms": 60 * 10 ** 9, "us": 5 * 10 ** 7, "ns": 5 * 10 ** 4}


@pytest.mark.parametrize("unit", TB.UNITS)
def test_every_resolution_and_unit(unit):
    from vaex_b200.frame import BinnerTime
    rng = np.random.default_rng(TB.UNITS.index(unit))
    for res in TB.UNITS:
        span = SPANS[res]
        if span is None or isinstance(span, tuple):
            lo, hi = span or ("1900-01-01", "2100-01-01")
            t = datetimes(rng, 3000, "ns" if unit in ("ms", "us", "ns") else "s", lo, hi).astype(f"M8[{unit}]")
            if span is None:
                t[:3] = np.array(["1900-02-28", "2000-02-29", "1969-12-31"], dtype="M8[D]").astype(t.dtype)
        else:
            # just before 1970-01-01: a unit coarser than the window puts every row in one tick, so the grid stays one period
            t = (rng.integers(-span, 0, 3000)).astype("M8[ns]").astype(f"M8[{unit}]")
        df = frame({"t": t}, "device")
        for every in (1, 3, 7) if res in ("M", "W", "D", "h") else (1,):
            out = df.groupby(BinnerTime("t", res, df=df, every=every), agg="count")
            keys, cells = expected_time(t, res, every)
            used, counts = grouped(cells, t, len)
            np.testing.assert_array_equal(out["t"], keys[used], err_msg=f"{unit} -> {res} every {every}")
            np.testing.assert_array_equal(out["count"], counts, err_msg=f"{unit} -> {res} every {every}")


def test_nat_masked_filter_and_selection():
    from vaex_b200 import agg as A
    from vaex_b200.frame import BinnerTime
    rng = np.random.default_rng(3)
    n = 10_000
    t = datetimes(rng, n, "s")
    t[::13] = np.datetime64("NaT")
    masked = rng.random(n) < 0.1
    x = rng.integers(-100, 100, n)
    tm = np.ma.array(t, mask=masked)
    # NaT and masked rows: the null group, never a key
    df = frame({"t": tm, "x": x})
    out = df.groupby(BinnerTime.per_week("t", df=df), agg={"c": A.count()})
    keys, cells = expected_time(t, "W", 1, masked=masked)
    used, counts = grouped(cells, x, len)
    np.testing.assert_array_equal(out["t"], keys[used])
    np.testing.assert_array_equal(out["c"], counts)
    # a filtered frame: the limits and the groups come from the rows that pass
    df = frame({"t": t, "x": x}, "device", filter="x > 20")
    out = df.groupby(BinnerTime.per_day("t", df=df), agg={"c": A.count()})
    keys, cells = expected_time(t, "D", 1, keep=x > 20)
    used, counts = grouped(cells, x, len)
    np.testing.assert_array_equal(out["t"], keys[used])
    np.testing.assert_array_equal(out["c"], counts)
    # a selection: a binned count over the time binner's spec counts the selected rows of every period
    df = frame({"t": t, "x": x}, "device")
    b = BinnerTime.per_year("t", df=df)
    grid = df.count(binby=[b.spec(df)], selection="x < 0", edges=True)
    _, cells = expected_time(t, "Y", 1)
    assert len(grid) == b.N + 2
    np.testing.assert_array_equal(grid[:b.N], np.bincount(cells[(cells >= 0) & (x < 0)], minlength=b.N))
    assert grid[b.N] == ((cells < 0) & (x < 0)).sum()


def test_nat_is_left_out_of_the_limits():
    """deviation: the reference's float32 minmax counts NaT as -2^63 and its BinnerTime breaks; here NaT is left out"""
    from vaex_b200.frame import BinnerTime
    t = np.array(["2020-01-05", "NaT", "2020-03-01"], dtype="M8[D]")
    df = frame({"t": t})
    b = BinnerTime.per_month("t", df=df)
    assert b.tmin == np.datetime64("2020-01-05") and b.N == 3
    out = df.groupby(b, agg="count")
    assert out["t"].tolist() == list(np.array(["2020-01", "2020-03"], dtype="M8[M]").tolist()) and out["count"].tolist() == [1, 1]


def test_ns_limits_keep_the_float32_rounding():
    """a ns minimum just before midnight rounds (float32, steps of about two minutes) past midnight: the reference's first day is the
    next one and the row before it falls out of range, as here"""
    from vaex_b200.frame import BinnerTime
    t = np.array(["2021-06-01T23:59:59.999", "2021-06-02T10:00", "2021-06-03T10:00"], dtype="M8[ns]")
    df = frame({"t": t}, "device")
    b = BinnerTime.per_day("t", df=df)
    tmin = reference_limits(t, np.ones(3, bool))[0]
    assert b.tmin == tmin and tmin.astype("M8[D]") == np.datetime64("2021-06-02")
    out = df.groupby(b, agg="count")
    assert out["t"].tolist() == np.array(["2021-06-02", "2021-06-03"], dtype="M8[D]").tolist() and out["count"].tolist() == [1, 1]


def test_mixed_keys():
    from vaex_b200 import agg as A
    from vaex_b200.frame import Binner, BinnerTime
    rng = np.random.default_rng(5)
    n = 5000
    t = datetimes(rng, n, "D", "2020-01-01", "2021-01-01")
    s = np.array([f"k{v}" for v in rng.integers(0, 4, n)], dtype=object)
    g = rng.integers(0, 3, n)
    x = rng.uniform(-1, 11, n)
    df = frame({"t": t, "s": s, "g": g, "x": x}, "device")
    out = df.groupby([BinnerTime.per_month("t", df=df), "s"], agg={"c": A.count()}, sort=True)
    keys, cells = expected_time(t, "M", 1)
    got = sorted(zip(out["t"].tolist(), np.asarray(out["s"], dtype=object).tolist(), out["c"].tolist()))
    want = {}
    for c, sv in zip(cells, s):
        want[(keys[c].tolist(), sv)] = want.get((keys[c].tolist(), sv), 0) + 1
    assert got == sorted((a, b, v) for (a, b), v in want.items())
    out = df.groupby([Binner("x", 0, 10, 5, df=df), "g"], agg={"m": A.sum("g")}, sort=True)
    b = np.floor(x / 2).astype(int)
    ok = (x >= 0) & (x < 10)
    want = sorted({(1 + 2 * bb, gg) for bb, gg in zip(b[ok], g[ok])})
    assert sorted(zip(out["x"].tolist(), out["g"].tolist())) == [(float(a), b_) for a, b_ in want]
    with pytest.raises(NotImplementedError, match="Binner"):
        df.groupby([Binner("x", 0, 10, 5, df=df), "g"], agg="count", combine=True)
    with pytest.raises(NotImplementedError, match="BinnerTime"):
        df.groupby([BinnerTime.per_month("t", df=df), "g"], agg="count", combine=True)
    auto = df.groupby([Binner("x", 0, 10, 5, df=df), "g"], agg="count", combine="auto")
    assert auto["count"].sum() == ok.sum()


@pytest.mark.parametrize("ascending", [True, False])
@pytest.mark.parametrize("dropmissing", [False, True])
def test_binner_integer(ascending, dropmissing):
    from vaex_b200 import agg as A
    from vaex_b200.frame import BinnerInteger
    rng = np.random.default_rng(7)
    n = 4000
    g = rng.integers(-5, 25, n)  # values outside [0, 19] join the null group
    mask = rng.random(n) < 0.05
    x = rng.integers(0, 100, n)
    df = frame({"g": np.ma.array(g, mask=mask), "x": x})
    b = BinnerInteger("g", min_value=0, max_value=19, sort=True, ascending=ascending, dropmissing=dropmissing, df=df)
    out = df.groupby(b, agg={"s": A.sum("x")})
    null = mask | (g < 0) | (g > 19)
    order = list(range(20)) if ascending else list(range(19, -1, -1))
    want_keys = [v for v in order if ((g == v) & ~null).any()]
    want = [int(x[(g == v) & ~null].sum()) for v in want_keys]
    if not dropmissing:
        want_keys.append(None)
        want.append(int(x[null].sum()))
    assert isinstance(out["g"], np.ma.MaskedArray)
    assert out["g"].tolist() == want_keys and out["s"].tolist() == want
    with pytest.raises(TypeError):
        BinnerInteger("x", df=df)


def test_errors():
    from vaex_b200 import superagg
    from vaex_b200.frame import BinnerTime
    df = frame({"t": np.array(["2300-01-01", "2300-02-01"], dtype="M8[D]")})
    with pytest.raises(ValueError, match="overflows"):
        BinnerTime("t", "ns", df=df)
    with pytest.raises(ValueError, match="cells"):
        BinnerTime("t", "ns", df=frame({"t": np.array(["1990-01-01", "2000-01-01"], dtype="M8[D]")}))
    with pytest.raises(ValueError, match="multiplier"):
        BinnerTime("t", "D", df=frame({"t": np.arange(3).astype("M8[5s]")}))
    with pytest.raises(TypeError):
        BinnerTime("t", "D", df=frame({"t": np.arange(3)}))
    # the library refuses a bad time binner with its argument error
    grid = superagg.Grid([superagg.BinnerTime_int64(1, "t", "D", "D", 0, 3, 0)])
    agg = superagg.AggCount_int64(grid, 1, 1)
    grid.binners[0].set_data(0, np.arange(3, dtype=np.int64))
    with pytest.raises(Exception, match="every"):
        grid.bin(0, [agg], 3)


def test_1e8_rows_against_numpy():
    import torch
    from vaex_b200 import agg as A
    from vaex_b200.frame import BinnerTime
    n = 10 ** 8
    g = torch.Generator(device="cuda").manual_seed(0)
    lo = int(np.datetime64("2000-01-01", "ns").astype(np.int64))
    span = int(np.datetime64("2024-01-01", "ns").astype(np.int64)) - lo
    tt = torch.randint(0, span, (n,), device="cuda", generator=g, dtype=torch.int64) + lo
    y = torch.randint(0, 1000, (n,), device="cuda", generator=g, dtype=torch.int64)
    from vaex_b200.frame import Frame
    df = Frame({"t": DeviceDatetime(tt, "M8[ns]"), "y": y})
    out = df.groupby(BinnerTime.per_month("t", df=df), agg={"y": "sum"})
    t = tt.cpu().numpy().view("M8[ns]")
    keys, cells = expected_time(t, "M", 1)
    used = np.unique(cells[cells >= 0])
    ys = y.cpu().numpy()
    want = np.zeros(cells.max() + 1, np.int64)
    np.add.at(want, cells[cells >= 0], ys[cells >= 0])
    np.testing.assert_array_equal(out["t"], keys[used])
    np.testing.assert_array_equal(out["y_sum"], want[used])


def profiled_kernels():
    """the CUDA kernels of one groupby over a per-day time key on device columns, as torch.profiler records them"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from vaex_b200.frame import BinnerTime
    rng = np.random.default_rng(11)
    t = datetimes(rng, 1 << 20)
    df = frame({"t": t, "y": rng.standard_normal(1 << 20).astype(np.float32)}, "device")
    b = BinnerTime.per_day("t", df=df)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        df.groupby(b, agg={"y": "sum"})
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})


def test_time_key_runs_in_k_binby():
    """the time key runs in the generic kernel, never in a float fast path.  The profiler runs in a process of its own: a profiler
    session leaves state behind in the process that profiles it, and the other tests that profile must not inherit it"""
    import json
    import subprocess
    code = f"import json, sys; sys.path.insert(0, {HERE!r}); import test_gpu_groupby_binners as T; print(json.dumps(T.profiled_kernels()))"
    out = subprocess.run([sys.executable, "-c", code], cwd=os.path.dirname(HERE), capture_output=True, text=True, check=True).stdout
    names = json.loads(out.strip().splitlines()[-1])
    assert any("k_binby" in k for k in names), names
    assert not any(("k_ring" in k or "k_fast" in k or "k_tile" in k) for k in names), names
