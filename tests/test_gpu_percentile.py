"""percentile_approx / median_approx on the device: the finish kernels (csrc/percentile.cu) against the reference's own finish on the
golden grids, bit for bit, and Frame.percentile_approx end to end against the numpy restatement (tests/percentile_oracle.py) applied
to the C oracle's count grid."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import percentile_oracle as PO  # noqa: E402
from helpers import same_bits  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"]


def device_grid(counts):
    """a count grid (binby axes first, percentile axis last) in the device layout: first dimension fastest"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(counts.reshape(-1, order="F"))).cuda()


def test_golden_grids_bit_identical():
    from vaex_b200 import percentile as _pct
    cases = PO.load_golden()
    assert len(cases) >= 25
    for name, c in cases.items():
        g = device_grid(c["counts"])
        got = _pct.finish(g.data_ptr(), c["counts"].shape, c["limit"], c["percentage"])
        assert type(got).__name__ == c["result_type"], name
        assert same_bits(np.asarray(got), c["result"]), name


def test_device_output_and_long_percentage_lists():
    """more percentages than one launch takes, the result written to device memory"""
    import torch
    from vaex_b200 import percentile as _pct
    rng = np.random.default_rng(3)
    counts = rng.integers(0, 9, (40 + 3, 30 + 3, 100 + 3)).astype(np.int64)
    pct = [1, 5.5, 10, 20, 25, 30, 40, 50, 60, 70.25, 75, 80, 90, 99]
    out = torch.empty((len(pct), 40 * 30), dtype=torch.float64, device="cuda")
    _pct.grid_percentile(device_grid(counts).data_ptr(), counts.shape, -1.0, 2.0, pct, out=out)
    want = PO.finish_one(counts, [-1.0, 1.0], pct)
    assert same_bits(out.cpu().numpy().reshape((len(pct), 40, 30), order="F"), want)


def column(rng, dtype, n):
    if dtype == "bool":
        return rng.random(n) < 0.3
    if dtype.startswith("float"):
        a = (rng.standard_normal(n) * 10).astype(dtype)
        a[rng.random(n) < 0.01] = np.nan
        return a
    lo = max(np.iinfo(dtype).min, -60)
    return rng.integers(lo, 61, n).astype(dtype)


def oracle_count(cols, binby, limits, shape, expression, limit, P, selection=None):
    """count(*) over binby + [expression] with edges from the C oracle; `cols` are host arrays (numpy.ma for masked columns)"""
    from oracle import oracle as O

    def binner(name, lim, bins):
        a = cols[name]
        mask = np.ma.getmaskarray(a).astype(np.uint8) if np.ma.isMaskedArray(a) else None
        return O.scalar(np.ascontiguousarray(np.ma.getdata(a)), lim[0], lim[1], bins, mask=mask)
    binners = [binner(b, lim, s) for b, lim, s in zip(binby, limits, shape)] + [binner(expression, limit, P)]
    sel = None if selection is None else np.ascontiguousarray(selection).astype(np.uint8)
    return O.binby(binners, [O.agg("count", None, mask=sel)])[0]


def make_frame(cols, place, nthreads=3, filter=None):
    import torch
    from vaex_b200 import execution, frame
    if place == "device":
        cols = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in cols.items()}
    ex = execution.Executor(nthreads, chunk_size=None if place == "device" else 60_000)
    return frame.Frame(cols, executor=ex, pin=place == "pinned", filter=filter)


@pytest.mark.parametrize("i,dtype", list(enumerate(DTYPES)))
def test_percentile_approx_end_to_end(i, dtype):
    """every column dtype as the expression, 0-3 binby dimensions, masked values and NaN, host / device / pinned columns"""
    rng = np.random.default_rng(100 + i)
    n = 200_003
    nd = i % 4
    place = ["host", "device", "pinned"][i % 3]
    if place == "device" and (dtype.startswith("uint") or dtype == "bool"):
        place = "pinned"  # unsigned and bool columns stay on the host here (torch has no CUDA copy for most unsigned types)
    cols = {"v": column(rng, dtype, n)}
    for d in range(nd):
        cols[f"b{d}"] = rng.standard_normal(n).astype("f4" if d % 2 else "f8")
    if place != "device" and i % 2:
        cols["v"] = np.ma.array(cols["v"], mask=rng.random(n) < 0.05)
    binby = [f"b{d}" for d in range(nd)]
    limits = [[-2.5, 2.5]] * nd
    shape = [9, 6, 4][:nd]
    P = [64, 300, 17, 1024][i % 4]
    pct = [[10, 50, 90], 50, [25.0, 50.5], [33, 66.0]][i % 4]
    plim = [0.0, 1.0] if dtype == "bool" else "minmax"  # numpy cannot subtract bools: the reference fails there too
    f = make_frame(cols, place)
    try:
        got = f.percentile_approx("v", pct, binby=binby or None, limits=limits or None, shape=shape, percentile_shape=P, percentile_limits=plim)
        limit = f.minmax("v") if plim == "minmax" else plim
        grid = oracle_count(cols, binby, limits, shape, "v", limit, P)
        assert np.array_equal(f.count(binby=binby + ["v"], limits=limits + [list(limit)], shape=shape + [P], edges=True), grid)
        want = PO.percentile_approx([grid], [limit], pct, False)
        assert type(got) is type(want) and same_bits(np.asarray(got), np.asarray(want))
        if nd == 0:
            assert same_bits(np.asarray(f.median_approx("v", percentile_limits=plim)),
                             np.asarray(PO.percentile_approx([oracle_count(cols, [], [], [], "v", limit, 256)], [limit], 50, False)))
    finally:
        if f._pinned is not None:
            f._pinned.release()  # the columns are freed after the test: they must not stay registered


def test_lists_of_expressions_and_percentages_one_pass():
    rng = np.random.default_rng(8)
    n = 150_000
    cols = {"x": rng.standard_normal(n), "y": rng.standard_normal(n).astype("f4"), "b": rng.uniform(-1, 1, n)}
    f = make_frame(cols, "host")
    passes = f.executor.passes
    pl = [[-3.0, 3.0], [-2.0, 2.5]]
    got = f.percentile_approx(["x", "y"], [25, 50.0, 75], binby="b", limits=[-1, 1], shape=16, percentile_shape=200, percentile_limits=pl)
    assert f.executor.passes == passes + 1
    grids = [oracle_count(cols, ["b"], [[-1, 1]], [16], e, lim, 200) for e, lim in zip(["x", "y"], pl)]
    want = PO.percentile_approx(grids, pl, [25, 50.0, 75], True)
    assert got.shape == (2, 3, 16) and same_bits(got, want)
    # without binby, 0 and 100 return the limits themselves
    got = f.percentile_approx(["x", "y"], [0, 50, 100], percentile_limits=pl, percentile_shape=100)
    grids = [oracle_count(cols, [], [], [], e, lim, 100) for e, lim in zip(["x", "y"], pl)]
    assert same_bits(got, PO.percentile_approx(grids, pl, [0, 50, 100], True))
    with pytest.raises(ValueError):
        f.percentile_approx("x", [0, 50], binby="b", limits=[-1, 1], shape=4)  # numpy's inhomogeneous shape, as in the reference


@pytest.mark.parametrize("place", ["host", "device"])
def test_selection_and_filtered_frame(place):
    rng = np.random.default_rng(21)
    n = 180_000
    cols = {"x": rng.standard_normal(n), "y": rng.standard_normal(n).astype("f4"), "z": rng.standard_normal(n)}
    kw = dict(binby=["x", "y"], limits=[[-1, 2], [-2, 2]], shape=[8, 5], percentile_shape=128, selection="y > 0")
    f = make_frame(cols, place, filter="x > -1")
    got = f.percentile_approx("z", [20, 80], percentile_limits=[-3.0, 3.0], **kw)
    keep = cols["x"] > -1
    kept = {k: v[keep] for k, v in cols.items()}
    grid = oracle_count(kept, ["x", "y"], [[-1, 2], [-2, 2]], [8, 5], "z", [-3.0, 3.0], 128, selection=kept["y"] > 0)
    assert same_bits(got, PO.percentile_approx([grid], [[-3.0, 3.0]], [20, 80], False))
    # "minmax" limits take the selection into account
    f = make_frame(cols, place)
    got = f.percentile_approx("z", [20, 80], **kw)
    limit = f.minmax("z", selection="y > 0")
    grid = oracle_count(cols, ["x", "y"], [[-1, 2], [-2, 2]], [8, 5], "z", limit, 128, selection=cols["y"] > 0)
    assert same_bits(got, PO.percentile_approx([grid], [limit], [20, 80], False))
    # "minmax" limits take the selection into account
    f = make_frame(cols, place)
    got = f.percentile_approx("z", [20, 80], **kw)
    limit = f.minmax("z", selection="y > 0")
    grid = oracle_count(cols, ["x", "y"], [[-1, 2], [-2, 2]], [8, 5], "z", limit, 128, selection=cols["y"] > 0)
    assert same_bits(got, PO.percentile_approx([grid], [limit], [20, 80], False))


def test_known_answers():
    """tests/percentile_approx_test.py:28-37 of the reference, and the same at percentile_shape=65536"""
    from vaex_b200 import execution, frame
    for P in (256, 65536):
        low = frame.Frame({"x": np.array([0, 0, 10, 100, 200])}, executor=execution.Executor(1))
        high = frame.Frame({"x": np.array([0, 0, 90, 100, 200])}, executor=execution.Executor(1))
        assert low.median_approx("x", percentile_shape=P) < 10.
        assert high.median_approx("x", percentile_shape=P) > 90.


def test_limits_percentage():
    rng = np.random.default_rng(31)
    n = 250_000
    cols = {"x": rng.standard_normal(n).astype("f4"), "b": rng.uniform(0, 1, n)}
    f = make_frame(cols, "host")
    vmin, vmax = f.minmax("x")
    counts = oracle_count(cols, [], [], [], "x", (vmin, vmax), 16384)[2:-1]
    want = PO.limits_percentage(counts, vmin, vmax, 90)
    assert same_bits(f.limits("x", "90%"), want)
    assert same_bits(f.limits_percentage("x", 90), want)
    assert same_bits(np.asarray(f.limits(["x", "b"], ["90%", [0, 1]])[0]), want)
    got = f.percentile_approx("x", [10, 50.0], percentile_limits="99%", percentile_shape=512)
    limit = PO.limits_percentage(counts, vmin, vmax, 99)
    assert same_bits(got, PO.percentile_approx([oracle_count(cols, [], [], [], "x", limit, 512)], [limit], [10, 50.0], False))


def test_categorical_and_datetime_columns_raise():
    from vaex_b200 import execution, frame
    f = frame.Frame({"c": np.arange(10) % 3, "t": np.arange(10).astype("datetime64[s]"), "x": np.arange(10.)}, executor=execution.Executor(1))
    f.categorize("c")
    with pytest.raises(NotImplementedError, match="'c'"):
        f.percentile_approx("x", binby="c")
    with pytest.raises(NotImplementedError, match="'t'"):
        f.percentile_approx("t")


def test_scale_1e8_rows_2d():
    import torch
    from vaex_b200 import execution, frame
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    cols = {k: torch.randn(n, device="cuda", dtype=torch.float32, generator=g) for k in ("x", "y", "z")}
    f = frame.Frame(cols, executor=execution.Executor(1))
    kw = dict(binby=["x", "y"], limits=[[-3, 3]] * 2, shape=128)
    got = f.percentile_approx("z", [25, 50, 75], percentile_limits=[-4, 4], percentile_shape=1024, **kw)
    grid = f.count(binby=["x", "y", "z"], limits=[[-3, 3]] * 2 + [[-4, 4]], shape=[128, 128, 1024], edges=True)
    assert grid.sum() == n
    assert got.shape == (3, 128, 128) and same_bits(got, PO.percentile_approx([grid], [[-4, 4]], [25, 50, 75], False))


# ---- kernel choice: recorded with torch.profiler in a fresh process (late in a long pytest process its sessions can come back empty)
def _kernel_cases():
    """name -> (binby dimensions, percentile_shape, the kernel the host should choose)"""
    return {"2d_128": (2, 1024, "k_pct_cell"), "1d_128": (1, 1024, "k_pct_block"), "none_65536": (0, 65536, "k_pct_block")}


def _record_kernels(path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from vaex_b200 import execution, frame
    rng = np.random.default_rng(2)
    n = 1_000_000
    cols = {k: torch.from_numpy(rng.standard_normal(n).astype("f4")).cuda() for k in ("x", "y", "z")}
    f = frame.Frame(cols, executor=execution.Executor(1))
    out = {}
    for name, (nd, P, _) in _kernel_cases().items():
        def run():
            return f.percentile_approx("z", [25, 50], binby=["x", "y"][:nd] or None, limits=[[-3, 3]] * nd or None, shape=128, percentile_shape=P,
                                       percentile_limits=[-4, 4])
        names = []
        for _ in range(3):  # a session now and then comes back without kernel records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if "k_pct_" in e.name]
            if names:
                break
        out[name] = names
    with open(path, "w") as fh:
        json.dump(out, fh)


@pytest.fixture(scope="module")
def kernels(tmp_path_factory):
    import subprocess
    out = tmp_path_factory.mktemp("prof") / "kernels.json"
    subprocess.check_call([sys.executable, os.path.abspath(__file__), str(out)], cwd=os.path.dirname(HERE))
    return json.loads(out.read_text())


@pytest.mark.parametrize("name", sorted(_kernel_cases()))
def test_kernel_choice(name, kernels):
    want = _kernel_cases()[name][2]
    assert kernels[name] and all(want in k for k in kernels[name]), kernels[name]


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _record_kernels(sys.argv[1])
