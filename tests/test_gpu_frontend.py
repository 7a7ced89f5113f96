"""Selections through the task parts and the Frame methods: a masked selection mask selects none of its masked rows in every task
part, selection=False means no selection in every method, and every method rejects a selection that is not boolean alike."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def masked_selection(seed=3):
    """1000 selected rows (v = 1), 1500 rows whose selection is True under its mask (v = 5), 500 unselected rows (v = 6)"""
    rng = np.random.default_rng(seed)
    data = np.repeat([True, True, False], [1000, 1500, 500])
    mask = np.repeat([False, True, False], [1000, 1500, 500])
    v = np.repeat([1.0, 5.0, 6.0], [1000, 1500, 500])
    order = rng.permutation(len(v))
    return np.ma.array(data[order], mask=mask[order]), v[order], np.full(len(v), 0.5)


def test_masked_selection_mask_in_every_task_part():
    from vaex_b200 import mode as _mode
    from vaex_b200 import statistic as _stat
    from vaex_b200 import taskpart
    sel, v, x = masked_selection()
    n = len(v)
    spec = {"binners": [{"binner-type": "scalar", "expression": "x", "dtype": "float64", "count": 1, "minimum": 0.0, "maximum": 1.0}],
            "aggregations": [{"aggregation": "count", "selection": "s"}, {"aggregation": "sum", "expressions": ["v"], "selection": "s"}],
            "dtypes": {"x": "float64", "v": "float64"}}
    part = taskpart.TaskPartAggregation.decode(None, spec, nthreads=1)
    part.process(0, 0, n, None, [sel, sel], [x, v])
    part.reduce([])
    count, total = part.get_result()
    assert count.tolist() == [1000] and total.tolist() == [1000.0]

    stat = taskpart.TaskPartStatistic(None, (), [], np.dtype("f8"), ["s"], _stat.OP_ADD1, [], [], [], False, False)
    stat.process(0, 0, n, None, [sel], [])
    assert stat.get_result().tolist() == [1000.0]

    # the mode of v over the selected rows is the bin of v = 1; counting the masked rows would make it the bin of v = 5
    mode = taskpart.TaskPartMode(None, (8, 1), ["v", "x"], [0.0, 0.0], [8.0, 1.0], _mode.centers(0.0, 8.0, 8), selection=True)
    mode.process(0, 0, n, None, [sel], [v, x])
    assert mode.get_result().tolist() == [1.5]


@pytest.mark.parametrize("place", ["host", "device"])
def test_selection_false_is_no_selection(place):
    import torch
    from vaex_b200.execution import Executor
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(5)
    cols = {"x": rng.normal(0, 1, 50_000), "v": rng.integers(-50, 50, 50_000).astype("i4")}
    if place == "device":
        cols = {k: torch.from_numpy(a).cuda() for k, a in cols.items()}
    df = Frame(cols, executor=Executor(nthreads=3, chunk_size=7_001))
    kw = dict(binby="x", limits=[-3, 3], shape=16)
    assert np.array_equal(df.count(selection=False), df.count())
    assert np.array_equal(df.count(selection=False, **kw), df.count(**kw))
    assert np.array_equal(df.sum("v", selection=False, **kw), df.sum("v", **kw))
    assert np.array_equal(df.mean("v", selection=False, **kw), df.mean("v", **kw), equal_nan=True)


@pytest.mark.parametrize("method", ["count", "cov", "percentile_approx", "mutual_information", "mode"])
def test_a_selection_must_be_boolean(method):
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(6)
    df = Frame({"x": rng.normal(0, 1, 1000), "y": rng.normal(0, 1, 1000)})
    call = {"count": lambda s: df.count(binby="x", limits=[-3, 3], shape=8, selection=s),
            "cov": lambda s: df.cov("x", "y", selection=s),
            "percentile_approx": lambda s: df.percentile_approx("x", selection=s),
            "mutual_information": lambda s: df.mutual_information("x", "y", selection=s),
            "mode": lambda s: df.mode("x", binby="y", selection=s)}[method]
    with pytest.raises(ValueError, match="^a selection must be a boolean expression$"):
        call("x + 1")
    call("x > 0")


def test_legacy_statistics_take_a_mask_array_as_selection():
    """cov, correlation and binned minmax resolve a selection like the binned statistics do: a boolean array is a mask"""
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(7)
    x, y = rng.normal(0, 1, 20_000), rng.normal(0, 1, 20_000)
    df = Frame({"x": x, "y": y})
    np.testing.assert_allclose(df.cov("x", "y", selection=x > 0), df.cov("x", "y", selection="x > 0"), rtol=1e-12)
    assert np.array_equal(df.minmax("y", binby="x", limits=[-3, 3], shape=4, selection=x > 0),
                          df.minmax("y", binby="x", limits=[-3, 3], shape=4, selection="x > 0"))
