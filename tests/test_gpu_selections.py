"""Named selections on the GPU (vaex_b200/selections.py, csrc/lasso.cu): the reference's selection_test.py cases without signals and
agg_test.py's selection cases as data, the device lasso against the compiled reference's golden vectors and the numpy restatement in
both loops, the geometric selections against numpy evaluating the reference's own text, select_non_missing over every kind of missing
value, selection=True through every selection= method, and the feeds: host, pinned and torch columns, filtered frames, several
threads, small chunks and chains longer than one program.  Masks are compared element for element."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import lasso_oracle as L  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(HERE, "golden", "lasso_golden.npz"))


def frame(columns, **kw):
    from vaex_b200.frame import Frame
    return Frame(columns, **kw)


def mask_of(df, selection=True):
    return df._selection(selection).evaluate()


def device_lasso(xs, ys, bx, by, banded):
    import torch
    from vaex_b200.selections import LassoPlan, _Lasso
    x = torch.from_numpy(np.ascontiguousarray(bx, np.float64)).cuda()
    y = torch.from_numpy(np.ascontiguousarray(by, np.float64)).cuda()
    return _Lasso(LassoPlan(xs, ys, banded=banded), x, y).chunk(0, 0, len(bx)).to_numpy()


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("banded", [False, True])
def test_lasso_golden(banded):
    cases = sorted({k.split("_")[0] for k in GOLDEN.files}, key=int)
    for k in cases:
        vx, vy, x, y, want = (GOLDEN[f"{k}_{f}"] for f in ("vx", "vy", "x", "y", "mask"))
        got = device_lasso(vx, vy, x, y, banded and len(vx) >= 1)
        assert np.array_equal(got, want), str(GOLDEN[f"{k}_name"])


@pytest.mark.parametrize("nvert", [3, 64, 1000, 10000])
def test_lasso_random_rows_both_loops(nvert):
    rng = np.random.default_rng(nvert)
    n = 10_000_000
    xs, ys = L.polygon(nvert, seed=nvert)
    bx, by = rng.uniform(-1.6, 1.6, n), rng.uniform(-1.6, 1.6, n)
    plain = device_lasso(xs, ys, bx, by, False)
    banded = device_lasso(xs, ys, bx, by, True)
    assert np.array_equal(plain, banded)
    k = 100_000 if nvert <= 1000 else 20_000
    assert np.array_equal(plain[:k], L.lasso(xs, ys, bx[:k], by[:k]))
    assert 0.05 < plain.mean() < 0.95


# ---- the reference's selection_test.py ------------------------------------------------------------------------------------------
def ref_df():
    """the columns of the reference's test frame these cases read: x = 0..9, y = x**2 and m = x with its last row masked"""
    x = np.arange(10, dtype="f8")
    m = np.ma.array(x.copy(), mask=x == 9)
    return frame({"x": x, "y": x ** 2, "m": m})


def test_selection_basics():
    from vaex_b200 import selections
    df = ref_df()
    total = df.sum("x")
    df.select("x > 5")
    df.select("x <= 5", name="inverse")
    counts = df.count("x", selection=["default", "inverse", "x > 5", "default | inverse"])
    assert np.array_equal(counts, [4, 6, 4, 10])
    df.select("x <= 1", name="inverse", mode="subtract")
    assert np.array_equal(df.count("x", selection=["default", "inverse"]), [4, 4])
    assert df.sum("x", selection=True) < total
    for mode in selections._select_functions.keys():
        df.select("x > 5")
        df.select("x > 5", mode)
        df.select(None)
        df.select("x > 5", mode)
    df.select("x > 5")
    total_subset = df.sum("x", selection=True)
    df.select_inverse()
    total_subset_inverse = df.sum("x", selection=True)
    df.select("x <= 5")
    assert total_subset_inverse == df.sum("x", selection=True)
    assert total_subset_inverse + total_subset == total
    df.select("x > 5")
    df.select("x <= 5", name="inverse")
    df.select_inverse(name="inverse")
    assert np.array_equal(df.count("x", selection=["default", "inverse"]), [4, 4])


def test_selection_history_sums():
    df = ref_df()
    total = df.sum("x")
    df.select("x > 5")
    s1 = df.sum("x", selection=True)
    df.select("x < 7", mode="and")
    s2 = df.sum("x", selection=True)
    assert s2 < s1 < total
    df.selection_undo()
    assert df.sum("x", selection=True) == s1
    df.selection_redo()
    assert df.sum("x", selection=True) == s2


def test_selection_serialize():
    from vaex_b200 import selections
    df = ref_df()
    e = selections.SelectionExpression("x > 5", None, "and")
    df.set_selection(e)
    total_subset = df.sum("x", selection=True)
    df.set_selection(selections.selection_from_dict(e.to_dict()))
    assert df.sum("x", selection=True) == total_subset
    lasso = selections.SelectionLasso("x", "y", [0, 10, 10, 0], [-1, -1, 100, 100], selections.SelectionExpression("x > 5", None, "and"), "and")
    df.set_selection(lasso)
    assert df.sum("x", selection=True) == total_subset


def test_lasso_reference_case():
    df = ref_df()
    df.select_lasso("x", "y", [-0.1, 5.1, 5.1, -0.1], [-0.1, -0.1, 4.1, 4.1])
    assert df.sum("x", selection=True) == 0 + 1 + 2
    assert df.sum("y", selection=True) == 0 + 1 + 4
    df.select_lasso("m", "y", [8 - 0.1, 9 + 0.1, 9 + 0.1, 8 - 0.1], [-0.1, -0.1, 1000, 1000])
    assert mask_of(df).tolist() == [False] * 8 + [True, False]  # row 9 lies inside but its m is masked
    assert df.sum("x", selection=True) == 8 and df.sum("y", selection=True) == 8 ** 2
    # a masked row stays unselected under mode="or" (the exclusion comes after the combine)
    df.select("x >= 0")
    df.select_lasso("m", "y", [8 - 0.1, 9 + 0.1, 9 + 0.1, 8 - 0.1], [-0.1, -0.1, 1000, 1000], mode="or")
    assert mask_of(df).tolist() == [True] * 9 + [False]


def test_selection_dependencies_with_named():
    x = np.arange(10)
    df = frame({"x": x, "y": x ** 2})
    df.select("x < 4", name="lt4")
    df.select("x > 1", name="gt1")
    df.select("lt4 & gt1", name="combined")
    assert df.sum("x", selection="combined") == 2 + 3
    df.select("x < 5", name="lt4")  # the names are looked up when the selection is used
    assert df.sum("x", selection="combined") == 2 + 3 + 4


def test_selection_with_filtered_frame():
    df = frame({"x": np.arange(10)}).filter("x != 4")
    df.add_virtual_column("y", "x * x")
    assert df.count("y", selection="y > 0") == 8
    df.select("y > 0")
    assert df.count("y", selection=True) == 8


# ---- agg_test.py's selection cases -----------------------------------------------------------------------------------------------
def test_agg_selection_cases():
    x = np.arange(10, dtype="f8")
    y = x ** 2
    df = frame({"x": x, "y": y})
    df.select("x < 5")
    assert df.sum("x", selection=True) == np.nansum(x[:5])
    assert np.array_equal(df.sum("x", selection=True, binby=["x"], limits=[0, 10], shape=2), [np.nansum(x[:5]), 0])
    assert np.array_equal(df.sum("y", selection=True, binby=["x"], limits=[0, 10], shape=2), [np.nansum(y[:5]), 0])
    assert np.array_equal(df.count("x", binby="x", limits=[0, 10], shape=10, selection=True), [1] * 5 + [0] * 5)
    assert np.allclose(df.correlation("x", "y", selection=True), np.corrcoef(x[:5], y[:5])[0, 1])
    assert np.array_equal(df.minmax("x", selection=True), [0, 4]) and np.array_equal(df.minmax("y", selection=True), [0, 16])
    assert df.mean("x", selection=True) == 2.0


# ---- selection=True through every selection= method -----------------------------------------------------------------------------
def test_selection_true_everywhere():
    rng = np.random.default_rng(3)
    n = 200_000
    df = frame({"x": rng.standard_normal(n), "y": rng.standard_normal(n), "i": rng.integers(0, 50, n)}, nthreads=3)
    df.executor.chunk_size = 30_000
    df.select_circle("x", "y", 0.1, -0.2, 1.1)
    df.select("i < 40", mode="and")
    text = "((((x - 0.1) * (x - 0.1)) + ((y - -0.2) * (y - -0.2))) <= 1.2100000000000002) & (i < 40)"
    want = mask_of(df, text)
    assert np.array_equal(mask_of(df), want)
    same = lambda a, b: np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)  # noqa: E731
    assert same(df.count(binby=["x", "y"], limits=[[-2, 2]] * 2, shape=32, selection=True),
                df.count(binby=["x", "y"], limits=[[-2, 2]] * 2, shape=32, selection=text))
    for method in ("min", "max"):
        assert same(getattr(df, method)("x", selection=True), getattr(df, method)("x", selection=text)), method
    for method in ("sum", "mean", "std"):  # float sums may add in another order
        assert np.isclose(getattr(df, method)("x", selection=True), getattr(df, method)("x", selection=text), rtol=1e-12, atol=0), method
    assert np.allclose(df.cov("x", "y", selection=True), df.cov("x", "y", selection=text), rtol=1e-9, atol=1e-12)
    assert np.isclose(df.correlation("x", "y", selection=True), df.correlation("x", "y", selection=text), rtol=1e-9)
    assert same(df.minmax("x", selection=True), df.minmax("x", selection=text))
    assert same(df.limits("x", "90%", selection=True), df.limits("x", "90%", selection=text))
    assert same(df.percentile_approx("x", 30, selection=True), df.percentile_approx("x", 30, selection=text))
    assert np.isclose(df.mutual_information("x", "y", selection=True), df.mutual_information("x", "y", selection=text), rtol=1e-9)
    kw = dict(binby="x", limits=[-2, 2], shape=8, mode_shape=50, mode_limits=[0, 50])
    assert same(df.mode("i", selection=True, **kw), df.mode("i", selection=text, **kw))
    assert df.selected_length() == int(want.sum())


def test_selection_true_without_default_names_it():
    df = frame({"x": np.arange(5.0)})
    with pytest.raises(KeyError, match="default"):
        df.sum("x", selection=True)


# ---- geometric selections against numpy on the reference's text --------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["f8", "f4", "i8"])
def test_geometric_selections(dtype):
    from vaex_b200 import selections
    rng = np.random.default_rng(5)
    x = (rng.standard_normal(100_000) * 3).astype(dtype)
    y = (rng.standard_normal(100_000) * 3).astype(dtype)
    df = frame({"x": x, "y": y})
    cases = [("box", lambda: df.select_box(["x", "y"], [(1.2345678, -0.5), (-1, 2.0000004)]),
              selections.box_text(["x", "y"], [(1.2345678, -0.5), (-1, 2.0000004)])),
             ("circle", lambda: df.select_circle("x", "y", 0.5, -1, 2), selections.circle_text("x", "y", 0.5, -1, 2).reference),
             ("circle <", lambda: df.select_circle("x", "y", 1, 1, 1.5, inclusive=False), selections.circle_text("x", "y", 1, 1, 1.5, False).reference),
             ("ellipse", lambda: df.select_ellipse("x", "y", 2, -1, 5, 1, 30), selections.ellipse_text("x", "y", 2, -1, 5, 1, 30).reference),
             ("ellipse <", lambda: df.select_ellipse("x", "y", 0, 0, 2, 6, 100, inclusive=False),
              selections.ellipse_text("x", "y", 0, 0, 2, 6, 100, inclusive=False).reference)]
    for name, select, reference_text in cases:
        select()
        with np.errstate(all="ignore"):
            want = eval(reference_text, {"x": x, "y": y})
        assert np.array_equal(mask_of(df), want), name


# ---- select_non_missing ---------------------------------------------------------------------------------------------------------
def test_select_non_missing():
    f = np.array([0.0, np.nan, 2.0, 3.0, np.nan, 5.0])
    m = np.ma.array([0, 1, 2, 3, 4, 5.0], mask=[0, 0, 1, 0, 0, 0])
    a = pa.array([1, None, 3, 4, 5, 6])
    o = np.array(["a", "b", None, "d", "e", None], dtype=object)
    df = frame({"f": f, "m": m, "a": a, "o": o})
    df.select_non_missing(column_names=["f"])
    assert mask_of(df).tolist() == [True, False, True, True, False, True]
    df.select_non_missing(column_names=["m"])
    assert mask_of(df).tolist() == [True, True, False, True, True, True]
    df.select_non_missing(column_names=["a"])
    assert mask_of(df).tolist() == [True, False, True, True, True, True]
    df.select_non_missing(column_names=["o"])
    assert mask_of(df).tolist() == [True, True, False, True, True, False]
    df.select_non_missing()
    assert mask_of(df).tolist() == [True, False, False, True, False, False]
    df.select_non_missing(drop_nan=False, column_names=["f", "m"])
    assert mask_of(df).tolist() == [True, True, False, True, True, True]
    df.select_non_missing(drop_masked=False, column_names=["f", "m"])
    assert mask_of(df).tolist() == [True, False, True, True, False, True]


# ---- feeds -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("feed", ["host", "pinned", "torch"])
def test_feeds_filtered_threads_and_small_chunks(feed):
    import torch
    rng = np.random.default_rng(11)
    n = 300_000
    x, y, z = rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), rng.standard_normal(n).astype("f4")
    xs, ys = L.polygon(80, seed=2)
    cols = {"x": x, "y": y, "z": z}
    if feed == "torch":
        cols = {k: torch.from_numpy(v).cuda() for k, v in cols.items()}
    df = frame(cols, nthreads=4, pin=feed == "pinned")
    try:
        df.executor.chunk_size = 17_000
        df.select_lasso("x", "y", xs, ys)
        df.select("z > -0.5", mode="and", name="default")
        want = L.lasso(xs, ys, x, y) & (z > -0.5)
        assert np.array_equal(mask_of(df), want)
        assert df.count(selection=True) == want.sum()
        assert np.isclose(df.sum("z", selection=True), z[want].astype("f8").sum(), rtol=1e-9)
        dff = df.filter("x > 0")
        assert dff.count(selection=True) == (want & (x > 0)).sum()
        assert np.array_equal(dff.count(selection=["default", "default", "z < 0"]), [(want & (x > 0)).sum()] * 2 + [((z < 0) & (x > 0)).sum()])
    finally:
        if df._pinned is not None:
            df._pinned.release()  # the host columns are freed after the test: they must not stay registered


def test_lasso_over_expressions_and_dtypes():
    rng = np.random.default_rng(2)
    n = 50_000
    a = rng.uniform(-2, 2, n).astype("f4")
    b = rng.integers(-2, 3, n)
    c = rng.uniform(-2, 2, n).astype(">f8")
    df = frame({"a": a, "b": b, "c": c})
    df.add_virtual_column("v", "a * 2")
    xs, ys = L.polygon(9, seed=1)
    df.select_lasso("v", "c", xs, ys)
    assert np.array_equal(mask_of(df), L.lasso(xs, ys, (a * 2).astype("f8"), c.astype("f8")))
    df.select_lasso("b", "a", xs, ys)
    assert np.array_equal(mask_of(df), L.lasso(xs, ys, b.astype("f8"), a.astype("f8")))


def test_chain_longer_than_one_program():
    rng = np.random.default_rng(4)
    n = 100_000
    cols = {f"c{k}": rng.standard_normal(n) for k in range(12)}
    df = frame(cols)
    want = np.ones(n, bool)
    for k in range(12):
        df.select(f"c{k} > -1.5", mode="and")
        want &= cols[f"c{k}"] > -1.5
    sel = df._selection(True)
    assert len(sel.programs) > 1
    assert np.array_equal(sel.evaluate(), want)
    assert df.count(selection=True) == want.sum()


def test_select_non_missing_over_more_than_eight_columns():
    rng = np.random.default_rng(6)
    n = 200_000
    cols = {f"f{k}": np.where(rng.random(n) < 0.01, np.nan, rng.standard_normal(n)) for k in range(12)}
    cols["m"] = np.ma.array(rng.standard_normal(n), mask=rng.random(n) < 0.02)
    cols["a"] = pa.array(np.where(rng.random(n) < 0.02, None, 1.0).tolist(), type=pa.float64())
    df = frame(cols)
    df.select_non_missing()
    assert len(df._selection(True).programs) >= 2
    want = np.ones(n, bool)
    for k in range(12):
        want &= ~np.isnan(cols[f"f{k}"])
    want &= ~np.ma.getmaskarray(cols["m"]) & ~cols["a"].is_null().to_numpy(zero_copy_only=False)
    assert np.array_equal(mask_of(df), want)
    assert df.count(selection=True) == want.sum()


def test_eight_input_step_after_a_previous_selection():
    rng = np.random.default_rng(8)
    n = 200_000
    cols = {f"c{k}": rng.standard_normal(n) for k in range(9)}
    df = frame(cols)
    df.select("c8 > 0")
    df.select(" & ".join(f"(c{k} > -1)" for k in range(8)), mode="and")
    want = cols["c8"] > 0
    for k in range(8):
        want &= cols[f"c{k}"] > -1
    assert np.array_equal(mask_of(df), want)
    assert df.count(selection=True) == want.sum()


@pytest.mark.parametrize("dtype", ["int64", "uint64"])
def test_lasso_integer_coordinates_above_2_53(dtype):
    """the device's astype('float64') of integers beyond 2^53 rounds like numpy's"""
    import torch
    rng = np.random.default_rng(9)
    n = 100_000
    base = 2 ** 53
    x = (base + rng.integers(0, 4096, n)).astype(dtype)
    y = (base + rng.integers(0, 4096, n)).astype(dtype)
    xs = [base + 100.0, base + 3000.0, base + 3000.0, base + 100.0]
    ys = [base + 7.0, base + 7.0, base + 2001.0, base + 2001.0]
    want = L.lasso(xs, ys, x, y)
    assert want.any() and not want.all()
    feeds = [{"x": x, "y": y}]
    if dtype == "int64":
        feeds.append({"x": torch.from_numpy(x).cuda(), "y": torch.from_numpy(y).cuda()})
    for cols in feeds:
        df = frame(cols)
        df.select_lasso("x", "y", xs, ys)
        assert np.array_equal(mask_of(df), want)
