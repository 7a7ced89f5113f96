"""mutual_information on the device: Frame.mutual_information against the reference's own results (golden) and the numpy restatement,
and the finish kernel b200_grid_mutual_information alone on synthetic count grids, held to the per-cell bound of DESIGN.md section 3."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import mutual_information_oracle as MO  # noqa: E402
from helpers import same_bits  # noqa: E402

pytestmark = pytest.mark.gpu


def native(col):
    if np.ma.isMaskedArray(col):
        return np.ma.array(np.ma.getdata(col).astype(col.dtype.newbyteorder("=")), mask=np.ma.getmaskarray(col))
    col = np.asarray(col)
    return col.astype(col.dtype.newbyteorder("="))


def make_frame(cols, place, nthreads=3, filter=None):
    import torch
    from vaex_b200 import execution, frame
    if place == "device":
        cols = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in cols.items()}
    ex = execution.Executor(nthreads, chunk_size=None if place == "device" else 700)
    return frame.Frame(cols, executor=ex, pin=place == "pinned", filter=filter)


def device_grid(counts):
    import torch
    return torch.from_numpy(np.ascontiguousarray(counts.reshape(-1, order="F"))).cuda()


def finish_on_device(counts, d, out=None):
    """b200_grid_mutual_information of a numpy grid with edges (MI axes first): the values shaped like the binby cells"""
    from vaex_b200 import mutual_information as _mi
    g = device_grid(counts)
    got = _mi.grid_mutual_information(g.data_ptr(), counts.shape, d, out=out)
    return got, g


def expected(counts, d):
    """(restatement, bound) per binby cell of a grid with edges, shaped like the binby cells"""
    inner = counts[tuple([slice(2, -1)] * counts.ndim)]
    cells = inner.shape[d:]
    want, tol = np.zeros(cells), np.zeros(cells)
    for index in np.ndindex(*cells):
        c = inner[(Ellipsis,) + index]
        want[index] = MO.mi_cell(c.astype(np.float64))
        tol[index] = MO.bound(c)
    return want, tol


def check_grid(counts, d):
    got, _ = finish_on_device(counts, d)
    want, tol = expected(counts, d)
    got = got.reshape(want.shape, order="F")
    assert np.all(np.abs(got - want) <= tol), (np.max(np.abs(got - want) - tol), counts.shape, d)
    return got, want


# ---- Frame.mutual_information against the golden vectors --------------------------------------------------------------
@pytest.mark.parametrize("place", ["host", "device", "pinned"])
def test_golden_through_frame(place):
    frames, cases = MO.load_golden()
    ran = 0
    for name, case in cases.items():
        columns = {k: native(v) for k, v in frames[case["frame"]].items()}
        kwargs = case["kwargs"]
        if place == "device" and (case["frame"] == "local" or "selection" in kwargs):
            continue  # masked columns and the boolean selection column stay on the host (pinned covers them)
        f = make_frame(columns, place, filter=case["filter"])
        try:
            if "error" in case:
                with pytest.raises(Exception) as info:
                    f.mutual_information(**kwargs)
                assert type(info.value).__name__ == case["error"], name
                continue
            got = f.mutual_information(**kwargs)
            kept = columns
            if case["filter"]:
                keep = np.asarray(columns[case["filter"]], bool)
                kept = {k: v[keep] for k, v in columns.items()}
            assert type(got).__name__ == case["result_type"], name
            want = case["result"]
            tol = MO.mutual_information(kept, per_cell=MO.bound, **kwargs)
            if isinstance(got, tuple):
                got, labels = got
                assert [list(v) if isinstance(v, tuple) else v for v in labels] == case["labels"], name
                tol = np.max(tol[0])  # the values are sorted: one bound for all
            assert got.shape == want.shape, name
            assert np.all(np.abs(got - want) <= tol), (name, got, want, tol)
            ran += 1
        finally:
            if f._pinned is not None:
                f._pinned.release()
    assert ran >= (20 if place == "device" else 34)


def test_known_answer_on_the_filtered_frame():
    """reference tests/agg_test.py:443-447: 2.043192 at mi_shape=32 on df_local, which is filtered to 0 <= x < 10"""
    frames, _ = MO.load_golden()
    cols = {k: native(v) for k, v in frames["local"].items()}
    f = make_frame(cols, "host", filter="(x >= 0) & (x < 10)")
    limits = [list(f.minmax("x")), list(f.minmax("y"))]
    got = f.mutual_information("x", "y", mi_limits=limits, mi_shape=32)
    assert isinstance(got, np.ndarray) and got.shape == ()
    np.testing.assert_array_almost_equal(got, 2.043192)


# ---- the finish kernel alone on synthetic grids -------------------------------------------------------------------------
def random_grid(rng, mshape, bshape, high=50, zero=0.3):
    shape = tuple(m + 3 for m in mshape) + tuple(n + 3 for n in bshape)
    g = rng.integers(0, high, shape).astype(np.int64)
    g[rng.random(shape) < zero] = 0
    return g


@pytest.mark.parametrize("d", [1, 2, 3, 4])
@pytest.mark.parametrize("nb", [0, 1, 2, 3])
def test_kernel_random_grids(d, nb):
    rng = np.random.default_rng(10 * d + nb)
    mshape = {1: [33], 2: [7, 2], 3: [5, 1, 11], 4: [3, 2, 4, 2]}[d]
    bshape = [4, 3, 5][:nb]
    got, _ = check_grid(random_grid(rng, mshape, bshape), d)
    if d == 1:
        assert np.all(got == 0.0)


@pytest.mark.parametrize("mshape,bshape", [((1, 1), (6,)), ((2, 2), (300,)), ((1, 9), ()), ((2, 7), (17, 19)), ((255, 257), ()),
                                           ((256, 256), ()), ((256, 256), (5,)), ((253, 253), (16, 16)), ((32, 32), (64, 64)),
                                           ((64, 64, 64), ()), ((3,), (400,)), ((6096, 40), ()), ((6097, 40), (2,))])
def test_kernel_shapes_on_both_sides_of_the_switch(mshape, bshape):
    rng = np.random.default_rng(sum(mshape) + sum(bshape))
    check_grid(random_grid(rng, mshape, bshape, high=1000, zero=0.5), len(mshape))


def test_kernel_totals_past_2_53():
    rng = np.random.default_rng(53)
    for mshape, bshape in [((9, 13), (3,)), ((64, 64), ()), ((5, 6), (20, 20))]:
        g = random_grid(rng, mshape, bshape, zero=0.2)
        big = rng.random(g.shape) < 0.5
        g[big] = rng.integers(2**48, 2**52, int(big.sum()))
        inner = g[tuple([slice(2, -1)] * g.ndim)]
        assert inner.reshape(int(np.prod(mshape)), -1).sum(0).max() > 2**53  # per binby cell, below 2^63
        check_grid(g, len(mshape))


def test_kernel_exact_zeros_and_closed_forms():
    """one bin holding every row, exact outer products (MI 0 in exact arithmetic), a diagonal (MI = the entropy), empty cells"""
    rng = np.random.default_rng(7)
    for mshape, bshape in [((16, 16), ()), ((8, 8), (300,)), ((256, 256), ())]:
        nd = len(bshape)
        # one bin per cell: P = Q = 1
        g = np.zeros(tuple(m + 3 for m in mshape) + tuple(n + 3 for n in bshape), np.int64)
        g[(3, 5) + (slice(None),) * nd] = 12345
        got, _ = finish_on_device(g, 2)
        assert np.all(got == 0.0)
        # outer products a_i * b_j per cell
        a = rng.integers(1, 1000, (mshape[0],) + bshape)
        b = rng.integers(1, 1000, (mshape[1],) + bshape)
        g[...] = 0
        g[(slice(2, -1), slice(2, -1)) + (slice(2, -1),) * nd] = a[:, None] * b[None, :]
        got, want = check_grid(g, 2)
        _, tol = expected(g, 2)
        assert np.all(np.abs(got) <= tol)
        # a diagonal: MI = -Σ p log p
        g[...] = 0
        diag = rng.integers(1, 10**6, mshape[0])
        for j in range(mshape[0]):
            g[(j + 2, j + 2) + (slice(2, -1),) * nd] = diag[j]
        p = diag / diag.sum()
        got, _ = check_grid(g, 2)
        assert np.all(np.abs(got - (-np.sum(p * np.log(p)))) <= expected(g, 2)[1])
    # empty binby cells give exactly 0.0; edge counts are ignored
    g = random_grid(rng, (10, 10), (7, 300))
    g[..., 4, :] = 0
    g[2:-1, 2:-1, 2:-1, 10] = 0
    got, _ = finish_on_device(g, 2)
    got = got.reshape((7, 300), order="F")
    assert np.all(got[2, :] == 0.0) and np.all(got[:, 8] == 0.0)


def test_kernel_writes_device_memory_and_is_deterministic():
    import torch
    rng = np.random.default_rng(11)
    for mshape, bshape in [((32, 32), (20, 20)), ((256, 256), ()), ((40, 40, 40), (2,))]:
        g = random_grid(rng, mshape, bshape, high=10**6)
        host1, _ = finish_on_device(g, len(mshape))
        host2, _ = finish_on_device(g, len(mshape))
        assert same_bits(host1, host2)
        out = torch.full((host1.size,), np.nan, dtype=torch.float64, device="cuda")
        finish_on_device(g, len(mshape), out=out)
        assert same_bits(out.cpu().numpy(), host1)


def test_kernel_rejects_bad_shapes():
    with pytest.raises(RuntimeError, match="axis 1 has 3 cells"):
        finish_on_device(np.zeros((5, 3, 4), np.int64), 2)


# ---- Frame: selections, filters, expressions, batching, memory -----------------------------------------------------------
def rows(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(n)
    return {"a": a, "b": a + rng.standard_normal(n), "c": rng.uniform(-2, 2, n), "w": rng.standard_normal(n).astype("f4")}


def assert_within(got, columns, **kwargs):
    want = MO.mutual_information(columns, **kwargs)
    tol = MO.mutual_information(columns, per_cell=MO.bound, **kwargs)
    assert got.shape == want.shape and np.all(np.abs(got - want) <= tol)


@pytest.mark.parametrize("place", ["host", "device"])
def test_selection_filter_and_expression(place):
    cols = rows(120_000, 4)
    kw = dict(mi_shape=[24, 17], binby=["c"], shape=5, limits=[-2, 2])
    f = make_frame(cols, place, filter="a > -1")
    got = f.mutual_information(["a", "b", "w"], selection="c > 0", **kw)
    keep = cols["a"] > -1
    kept = {k: v[keep] for k, v in cols.items()}
    kept["s"] = kept["c"] > 0
    assert_within(got, kept, x=["a", "b", "w"], selection="s", **kw)
    f = make_frame(cols, place)
    got = f.mutual_information("a + b", "c", mi_shape=40)
    assert_within(got, dict(cols, **{"a + b": cols["a"] + cols["b"]}), x="a + b", y="c", mi_shape=40)


def test_batches_share_passes_under_a_lowered_budget(monkeypatch):
    from vaex_b200 import mutual_information as _mi
    cols = rows(200_000, 5)
    f = make_frame(cols, "host")
    kw = dict(x=["a", "b", "c"], mi_shape=64, mi_limits=[-4, 4])
    passes = f.executor.passes
    whole = f.mutual_information(**kw)
    assert f.executor.passes == passes + 1  # the six unique combinations in one pass
    monkeypatch.setattr(_mi, "GRID_BUDGET_BYTES", 2 * 67 * 67 * 8)
    passes = f.executor.passes
    batched = f.mutual_information(**kw)
    assert f.executor.passes == passes + 3
    assert same_bits(batched, whole)
    assert_within(whole, cols, **kw)


def test_limits_pre_pass_runs_once_per_name(monkeypatch):
    """x=[3 columns] has 6 unique pairs naming each column 4 times; with binby, every name's minmax runs once per call"""
    from vaex_b200 import frame
    cols = rows(50_000, 7)
    f = make_frame(cols, "host")
    calls = []
    minmax = frame.Frame.minmax

    def counted(self, expression, *args, **kwargs):
        calls.append(expression)
        return minmax(self, expression, *args, **kwargs)
    monkeypatch.setattr(frame.Frame, "minmax", counted)
    got = f.mutual_information(["a", "b", "c"], mi_shape=16, binby=["w", "c"], shape=3)
    assert sorted(calls) == ["a", "b", "c", "w"]
    assert_within(got, cols, x=["a", "b", "c"], mi_shape=16, binby=["w", "c"], shape=3)
    calls.clear()
    f.mutual_information([["a", "b"], ["b", "c"]], mi_limits=[[[-4, 4], [-5, 5]], "minmax"], mi_shape=8)
    assert sorted(calls) == ["b", "c"]  # explicit pairs pass through


def test_a_grid_larger_than_the_device_raises_memory_error():
    cols = rows(1000, 6)
    f = make_frame(cols, "host")
    with pytest.raises(MemoryError, match=r"\(256, 256, 512, 512, 512\)"):
        f.mutual_information("a", "b", mi_limits=[-4, 4], binby=["c", "w", "a"], limits=[-2, 2], shape=512)


def test_scale_1e8_rows():
    import torch
    from vaex_b200 import execution, frame
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(n, device="cuda", dtype=torch.float32, generator=g)
    cols = {"x": x, "y": x + torch.randn(n, device="cuda", dtype=torch.float32, generator=g),
            "z": torch.randn(n, device="cuda", dtype=torch.float32, generator=g)}
    f = frame.Frame(cols, executor=execution.Executor(1))
    lim = [[-4, 4], [-6, 6]]
    got = f.mutual_information("x", "y", mi_limits=lim, mi_shape=256)
    counts = f.count(binby=["x", "y"], limits=lim, shape=256)
    assert counts.sum() > 0.99 * n
    assert abs(got - MO.mi_cell(counts.astype(np.float64))) <= MO.bound(counts)
    got = f.mutual_information("x", "y", mi_limits=lim, mi_shape=64, binby=["z"], limits=[-3, 3], shape=128)
    counts = f.count(binby=["x", "y", "z"], limits=lim + [[-3, 3]], shape=[64, 64, 128])
    want, tol = np.array([MO.mi_cell(counts[..., i].astype(np.float64)) for i in range(128)]), np.array([MO.bound(counts[..., i]) for i in range(128)])
    assert got.shape == (128,) and np.all(np.abs(got - want) <= tol)


# ---- kernel choice: recorded with torch.profiler in a fresh process -------------------------------------------------------
def _kernel_cases():
    """name -> (MI shape, binby shape, the kernel the host should choose)"""
    return {"cells_256_block_1225": ((32, 32), (16, 16), "k_mi_cell"), "cells_255": ((32, 32), (15, 17), "k_mi_marg"),
            "cells_256_block_65536": ((253, 253), (16, 16), "k_mi_cell"), "cells_256_block_67081": ((256, 256), (16, 16), "k_mi_marg"),
            "no_binby_256": ((256, 256), (), "k_mi_marg"), "dimension_3": ((64, 64, 64), (), "k_mi_marg"),
            "marginals_2049": ((2046, 3), (256,), "k_mi_marg")}


def _record_kernels(path):
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(2)
    out = {}
    for name, (mshape, bshape, _) in _kernel_cases().items():
        shape = tuple(m + 3 for m in mshape) + tuple(n + 3 for n in bshape)
        counts = rng.integers(0, 3, shape).astype(np.int64)
        names = []
        for _ in range(3):  # a session now and then comes back without kernel records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                finish_on_device(counts, len(mshape))
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if "k_mi_" in e.name]
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
    assert kernels[name] and any(want in k for k in kernels[name]), kernels[name]
    if want == "k_mi_cell":
        assert not any("k_mi_marg" in k for k in kernels[name])


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _record_kernels(sys.argv[1])
