"""The legacy statistics on the device (csrc/statistic.cu, taskpart.TaskPartStatistic, Frame.cov / correlation / covar / binned
minmax) against the numpy restatement tests/statistic_oracle.py, which tests/test_statistic_oracle_cpu.py pins bit for bit against the
compiled vaexfast.  Counts, min/max and FIRST must agree bit for bit (min/max up to the documented signed-zero rule); fp64 sums and
products within the recursive-summation bound, since the device adds in a different order."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

import statistic_cases  # noqa: E402
import statistic_oracle as SO  # noqa: E402
from helpers import same_bits  # noqa: E402

pytestmark = pytest.mark.gpu

EPS = 2.0**-53


def _sum_fields(op, nw):
    if op == SO.MOMENTS_01:
        return [1]
    if op == SO.MOMENTS_012:
        return [1, 2]
    if op == SO.COV:
        return list(range(nw, 2 * nw)) + list(range(2 * nw + nw * nw, 2 * nw + 2 * nw * nw))
    return []


def _abs_case(case):
    out = dict(case)
    out["weights"] = [np.ma.array(np.abs(np.ma.getdata(w).astype(np.float64)), mask=np.ma.getmaskarray(w)) if np.ma.isMaskedArray(w)
                      else np.abs(_native_f64(w)) for w in case["weights"]]
    return out


def _native_f64(a):
    a = np.asarray(a)
    return a.astype(a.dtype.newbyteorder("=")).astype(np.float64) if a.dtype.kind != "b" else a.astype(np.float64)


def assert_grid(got, want, case, mag=None):
    """counts / min / max / FIRST bit for bit; sums within n * eps * sum|terms| (recursive summation, both orders)"""
    op, nw = case["op"], len(case["weights"])
    assert got.shape == want.shape
    sums = _sum_fields(op, nw)
    exact = [f for f in range(got.shape[-1]) if f not in sums]
    g, w = got[..., exact], want[..., exact]
    if op == SO.MIN_MAX:  # the device orders -0.0 below +0.0; the reference keeps the zero that arrived first
        zero = (g == 0) & (w == 0)
        g, w = np.where(zero, 0.0, g), np.where(zero, 0.0, w)
    assert same_bits(g, w)
    if sums:
        if mag is None:
            mag = SO.process(**_abs_case(case))
        n = np.maximum(np.max(want[..., :nw if op == SO.COV else 1], axis=-1, keepdims=True), 1)  # terms per cell, at most
        gs, ws, ms = got[..., sums], want[..., sums], mag[..., sums]
        nan = np.isnan(ws)
        assert np.array_equal(np.isnan(gs), nan)
        ok = ~nan & np.isfinite(ws)
        bound = 2 * (n + 2) * EPS * ms
        bound = np.broadcast_to(bound, ms.shape)
        assert np.all(np.abs(gs[ok] - ws[ok]) <= bound[ok] + 1e-300)
        assert same_bits(gs[~ok & ~nan], ws[~ok & ~nan])


def device_grid(case, chunk=None, to_device=False, slots=1):
    from vaex_b200 import statistic as ST
    import torch
    cols = list(case["binby"]) + list(case["weights"])
    n = len(cols[0])
    dtypes = [np.asarray(np.ma.getdata(c)).dtype for c in cols]
    cls = ST.compute_class(dtypes)
    st = ST.Statistic(case["op"], cls, case["sizes"], case["minima"], case["maxima"], case["edges"], len(case["weights"]), len(case["selections"]))
    chunk = chunk or n
    nd = len(case["binby"])
    keep = []
    for k, i1 in enumerate(range(0, n, chunk)):
        i2 = min(i1 + chunk, n)
        blocks = [c[i1:i2] for c in cols]
        sels = [None if s is None else s[i1:i2] for s in case["selections"]]
        if to_device:
            def dev(a):
                if np.ma.isMaskedArray(a) or a.dtype.byteorder not in "=|":
                    return a  # masked and byte-swapped blocks stay on the host: a MIXED call
                return torch.from_numpy(np.ascontiguousarray(a)).cuda()
            blocks = [dev(b) for b in blocks]
            sels = [None if s is None else torch.from_numpy(np.ascontiguousarray(s)).cuda() for s in sels]
        keep.append(st.bin(k % slots, blocks[:nd], blocks[nd:], sels, i2 - i1, row_offset=i1))
    out = st.read()
    st.close()
    return out


def test_golden_parity():
    from golden_statistic import cases
    g = np.load(os.path.join(HERE, "golden", "statistic_golden.npz"))
    for name, case in cases().items():
        assert_grid(device_grid(case), g[name], case)


@pytest.mark.parametrize("seed", range(40))
def test_random_parity(seed):
    rng = np.random.default_rng(1000 + seed)
    case = statistic_cases.random_case(rng, n=int(rng.choice([3000, 70_001])))
    chunk = [None, 9_000][seed % 2]
    want = SO.process(**case, chunk=chunk)
    assert_grid(device_grid(case, chunk=chunk, to_device=seed % 3 == 0, slots=1 + seed % 3), want, case)


def test_one_row_cells_bit_exact():
    rng = np.random.default_rng(5)
    x = rng.uniform(0, 1, 64)
    w = [rng.standard_normal(64) for _ in range(3)]
    for op, weights in ((SO.MOMENTS_012, w[:1]), (SO.COV, w)):
        case = dict(binby=[x], weights=weights, selections=[None], op=op, sizes=[1 << 20], minima=[0.0], maxima=[1.0], edges=False)
        assert same_bits(device_grid(case), SO.process(**case))


def _kernels(fn):
    """names of the k_stat kernels `fn` launched.  A profiler session now and then comes back without its kernel records (seen on the
    first launch of a lazily loaded kernel), so `fn` must be repeatable: it runs again when that happens."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if "k_stat" in e.name and "k_stat_fill" not in e.name]
        if names:
            return names
    raise AssertionError("torch.profiler recorded no k_stat kernel")


STRATEGIES = ["reg", "smem", "global"]


def _strategy_case(strategy, op, dtype):
    """no binby and one selection -> k_stat_reg; a 16-cell grid with two selections -> k_stat_smem; 128^2 cells -> k_stat_global"""
    rng = np.random.default_rng(op * 10 + len(strategy))
    n = 200_003
    nw = {SO.ADD1: 1, SO.COV: 3, SO.FIRST: 2}.get(op, 1)
    cols = [statistic_cases.column(rng, dtype, n) for _ in range(2 + nw)]
    if strategy == "reg":
        binby, sizes, sels = [], [], [None]
    elif strategy == "smem":
        binby, sizes, sels = cols[:1], [16], [None, rng.random(n) < 0.5]
    else:
        binby, sizes, sels = cols[:2], [128, 128], [None]
    return dict(binby=binby, weights=cols[2:], selections=sels, op=op, sizes=sizes, minima=[-3.0] * len(sizes), maxima=[3.0] * len(sizes),
                edges=False)


@pytest.fixture(scope="module")
def strategy_kernels(tmp_path_factory):
    """the k_stat kernels every strategy case launched, recorded with torch.profiler in a fresh process: late in a long pytest process
    the profiler's sessions come back without kernel records more and more often"""
    import json
    import subprocess
    out = tmp_path_factory.mktemp("prof") / "kernels.json"
    subprocess.check_call([sys.executable, os.path.abspath(__file__), str(out)], cwd=os.path.dirname(HERE))
    return json.loads(out.read_text())


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("op", statistic_cases.OPS)
@pytest.mark.parametrize("strategy", STRATEGIES)
def test_every_strategy_class_and_op(strategy, op, dtype, strategy_kernels):
    names = strategy_kernels["%s-%d-%s" % (strategy, op, dtype)]
    want_kernel = "k_stat_first" if op == SO.FIRST else "k_stat_" + strategy
    assert names and all(want_kernel in k for k in names), names
    case = _strategy_case(strategy, op, dtype)
    assert_grid(device_grid(case, to_device=True), SO.process(**case), case)


def test_host_device_and_mixed_columns_agree():
    rng = np.random.default_rng(11)
    n = 300_000
    x = rng.standard_normal(n).astype("f4")
    w = [rng.standard_normal(n).astype("f4") for _ in range(2)]
    w[1] = np.ma.array(w[1], mask=rng.random(n) < 0.1)
    case = dict(binby=[x], weights=w, selections=[None, rng.random(n) < 0.3], op=SO.COV, sizes=[50], minima=[-2.0], maxima=[2.0], edges=True)
    want = SO.process(**case)
    for dev in (False, True):
        assert_grid(device_grid(case, chunk=64_000, to_device=dev, slots=3), want, case)


def _frame(cols, nthreads=4, filter=None):
    from vaex_b200 import execution, frame
    return frame.Frame(cols, executor=execution.Executor(nthreads, chunk_size=50_000), filter=filter)


def _finish_cov(values, N):
    counts, sums = values[..., :N], values[..., N:2 * N]
    with np.errstate(divide="ignore", invalid="ignore"):
        means = sums / counts
        shp = values.shape[:-1] + (N, N)
        return values[..., 2 * N + N**2:].reshape(shp) / values[..., 2 * N:2 * N + N**2].reshape(shp) - means[..., None] * means[..., None, :]


def test_frame_cov_correlation_covar_minmax():
    import torch
    rng = np.random.default_rng(3)
    n = 400_000
    x, y, z = rng.standard_normal(n), rng.standard_normal(n), rng.standard_normal(n).astype("f4")
    y = x * 0.5 + y
    cols = {"x": x, "y": y, "z": z}
    for c in (cols, {k: torch.from_numpy(v).cuda() for k, v in cols.items()}):
        df = _frame(c)
        want = _finish_cov(SO.process([], [x, y, z], [None], SO.COV, [], [], []), 3)[0]
        got = df.cov(["x", "y", "z"])
        assert np.allclose(got, want, rtol=1e-9, atol=1e-12)
        assert np.allclose(df.cov("x", "y"), _finish_cov(SO.process([], [x, y], [None], SO.COV, [], [], []), 2)[0], rtol=1e-9)
        corr = df.correlation(["x", "y", "z"])
        d = np.sqrt(np.diag(want))
        assert np.allclose(corr, want / np.outer(d, d), rtol=1e-9)
        assert np.isclose(df.correlation("x", "y"), corr[0, 1], rtol=1e-12)
        binned = df.cov("x", "y", binby="z", limits=[-2, 2], shape=8)
        wantb = _finish_cov(SO.process([z], [x, y], [None], SO.COV, [8], [-2.0], [2.0]), 2)[0]
        assert np.allclose(binned, wantb, rtol=1e-9, equal_nan=True)
        cv = df.covar("x", "y")
        assert np.isclose(cv, np.mean(x * y) - np.mean(x) * np.mean(y), rtol=1e-9)
        mm = df.minmax("x", binby="z", limits=[-2, 2], shape=8)
        wantm = SO.process([z], [x], [None], SO.MIN_MAX, [8], [-2.0], [2.0])[0]
        assert same_bits(mm, wantm)
    # a filtered frame and a list of selections
    df = _frame(cols, filter="z > 0")
    sel = ["x > 0", None]
    got = df.minmax("y", binby="x", limits=[-3, 3], shape=10, selection=sel)
    keep = z > 0
    want = SO.process([x[keep]], [y[keep]], [(x > 0)[keep], None], SO.MIN_MAX, [10], [-3.0], [3.0])
    assert same_bits(got, want)


def _exact_cov(cols):
    """cov[i][j] = sum(x_i x_j)/n - (sum x_i/n)(sum x_j/n) in exact rational arithmetic, and the same with |x| (the error scale)"""
    from fractions import Fraction
    n = len(cols[0])
    F = [[Fraction(float(v)) for v in c] for c in cols]
    N = len(cols)
    sums = [sum(f) for f in F]
    abss = [sum(abs(v) for v in f) for f in F]
    cov = [[None] * N for _ in range(N)]
    scale = [[None] * N for _ in range(N)]
    for i in range(N):
        for j in range(N):
            sxy = sum(a * b for a, b in zip(F[i], F[j]))
            axy = sum(abs(a * b) for a, b in zip(F[i], F[j]))
            cov[i][j] = sxy / n - (sums[i] / n) * (sums[j] / n)
            scale[i][j] = axy / n + (abss[i] / n) * (abss[j] / n)
    return cov, scale


def test_frame_finish_against_exact_arithmetic():
    """Frame.cov / correlation / covar against the reference's finish (dataframe.py:1461-1479, 1380-1387, 1272-1274) restated in
    exact rational arithmetic: the device result may differ by the rounding of n-term sums and of the finish itself"""
    rng = np.random.default_rng(21)
    n = 20_000
    x = rng.standard_normal(n) * 3 + 1
    y = 0.3 * x + rng.standard_normal(n)
    z = rng.standard_normal(n).astype("f4").astype("f8")
    df = _frame({"x": x, "y": y, "z": z}, nthreads=3)
    df.executor.chunk_size = 3_000
    from fractions import Fraction
    cov, scale = _exact_cov([x, y, z])
    got = df.cov(["x", "y", "z"])
    tol = lambda i, j: float(2 * (n + 8) * Fraction(EPS) * scale[i][j])  # noqa: E731
    for i in range(3):
        for j in range(3):
            assert abs(Fraction(float(got[i, j])) - cov[i][j]) <= Fraction(tol(i, j)), (i, j)
    corr = df.correlation(["x", "y", "z"])
    for i in range(3):
        for j in range(3):
            c = float(cov[i][j]) / np.sqrt(float(cov[i][i]) * float(cov[j][j]))
            rel = tol(i, j) / abs(float(cov[i][j])) + tol(i, i) / float(cov[i][i]) + tol(j, j) / float(cov[j][j]) + 8 * EPS
            assert abs(corr[i, j] - c) <= abs(c) * rel, (i, j)
    assert abs(Fraction(float(df.covar("x", "y"))) - cov[0][1]) <= Fraction(tol(0, 1))


def test_filtered_host_frame_many_threads_big_chunks():
    """host columns on a filtered Frame: every chunk is compacted into fresh device buffers on its worker's slot, while other
    workers' kernels (here k_stat_global, COV on a 128^2 grid) may still read theirs"""
    rng = np.random.default_rng(31)
    n = 16_000_000
    cols = {"a": rng.standard_normal(n).astype("f4"), "b": rng.standard_normal(n).astype("f4"), "u": rng.standard_normal(n),
            "v": rng.standard_normal(n), "f": rng.random(n).astype("f4")}
    from vaex_b200 import execution, frame, statistic as ST
    df = frame.Frame(cols, executor=execution.Executor(8, chunk_size=2_000_000), filter="f > 0.3")
    got = df._statistic(ST.OP_COV, ["a", "b"], ["u", "v"], [[-3, 3], [-3, 3]], 128, None)
    keep = cols["f"] > 0.3
    case = dict(binby=[cols["a"][keep], cols["b"][keep]], weights=[cols["u"][keep], cols["v"][keep]], selections=[None], op=SO.COV,
                sizes=[128, 128], minima=[-3.0, -3.0], maxima=[3.0, 3.0], edges=False)
    want = SO.process(**case)
    assert_grid(got[None], want, case)


def test_count_star_without_columns():
    """OP_ADD1 with no binby and no weight (the reference's `+= i2 - i1` / `np.sum(selection_mask)`, cpu.py:578-584)"""
    from vaex_b200 import taskpart, statistic as ST
    rng = np.random.default_rng(8)
    sel = rng.random(100_000) < 0.3
    p = taskpart.TaskPartStatistic(None, (), [], np.dtype("f8"), [None, "s"], ST.OP_ADD1, [], [], [], False, True)
    for t, i1 in enumerate(range(0, 100_000, 30_000)):
        i2 = min(i1 + 30_000, 100_000)
        p.process(t % 2, i1, i2, None, [None, sel[i1:i2]], [])
    assert np.array_equal(p.get_result(), [[100_000.0], [float(sel.sum())]])


@pytest.mark.parametrize("nw", [5, 7])
@pytest.mark.parametrize("sizes", [[], [9], [128, 40]])
def test_cov_more_than_four_weights(nw, sizes):
    """COV with more than four weights reads them per row (the NT = 0 variants), without binby too"""
    rng = np.random.default_rng(nw * 10 + len(sizes))
    n = 150_001
    dts = ["float32", "float64", "int32", "uint16", "int8", "float32", "float64"]
    cols = [statistic_cases.column(rng, dts[i % len(dts)], n) for i in range(len(sizes) + nw)]
    case = dict(binby=cols[:len(sizes)], weights=cols[len(sizes):], selections=[None, rng.random(n) < 0.5], op=SO.COV, sizes=sizes,
                minima=[-3.0] * len(sizes), maxima=[3.0] * len(sizes), edges=False)
    assert_grid(device_grid(case, chunk=40_000, to_device=True, slots=2), SO.process(**case, chunk=40_000), case)


@pytest.mark.parametrize("op", statistic_cases.OPS)
def test_unaligned_device_columns(op):
    """device columns that start off a 16-byte boundary take the scalar loads (StatParams.vec = 0)"""
    import torch
    from vaex_b200 import statistic as ST
    rng = np.random.default_rng(40 + op)
    n = 100_003
    nw = {SO.COV: 3, SO.FIRST: 2}.get(op, 1)
    cols = [statistic_cases.column(rng, dt, n + 1) for dt in ["float32", "float64", "int16", "float64"][:1 + nw]]
    case = dict(binby=[c[1:] for c in cols[:1]], weights=[c[1:] for c in cols[1:]], selections=[None], op=op, sizes=[33], minima=[-3.0],
                maxima=[3.0], edges=True)
    dev = [torch.from_numpy(c).cuda()[1:] for c in cols]
    assert all(t.data_ptr() % 16 for t in dev)
    cls = ST.compute_class([c.dtype for c in cols])
    st = ST.Statistic(op, cls, [36], [-3.0], [3.0], True, nw, 1)
    st.bin(0, dev[:1], dev[1:], [None], n, 0)
    got = st.read()
    st.close()
    case["sizes"] = [36]
    assert_grid(got, SO.process(**case), case)


def test_datetime_columns():
    """datetime weights and binby go through the float32 class like the reference's as_flat_array (the signed count of units)"""
    from vaex_b200 import taskpart, statistic as ST
    rng = np.random.default_rng(9)
    n = 50_000
    t = (rng.integers(-2**40, 2**60, n)).astype("M8[ns]")
    p = taskpart.TaskPartStatistic(None, (), [], np.dtype("f8"), [None], ST.OP_MIN_MAX, ["t"], [], [], False, False)
    p.process(0, 0, n, None, [None], [t])
    f = t.astype("f4").astype("f8")
    assert np.array_equal(p.get_result(), [f.min(), f.max()])
    lo, hi = float(f.min()), float(f.max())
    p = taskpart.TaskPartStatistic(None, (10,), ["t"], np.dtype("f8"), [None], ST.OP_ADD1, [], [lo], [hi], False, False)
    p.process(0, 0, n, None, [None], [t])
    want = SO.statistic_nd([t.astype("f4")], [], SO.init_grid(SO.ADD1, (10, 1)), [lo], [hi], SO.ADD1, False)
    assert np.array_equal(p.get_result(), want)


def test_legacy_statistic_spec_through_the_registry(monkeypatch):
    """TaskStatistic.encode's spec (vaex/tasks.py:409-413, '_op' encoding :375-394) decoded through a stub 'task-part-cpu' registry"""
    from vaex_b200 import statistic as ST, vaex_plugin
    registry, types_ = {}, {}
    vaex = types.ModuleType("vaex")
    cpu = types.ModuleType("vaex.cpu")

    def register(cls):
        types_[cls.snake_name] = cls
        return cls
    cpu.register = register
    for name in ("TaskPartAggregation", "TaskPartHashmapUniqueCreate", "TaskPartStatistic"):
        setattr(cpu, name, register(type(name, (), {"snake_name": {"TaskPartAggregation": "aggregations", "TaskPartHashmapUniqueCreate":
                                                                   "hash_map_unique_create", "TaskPartStatistic": "legacy_statistic"}[name]})))
    at = types.ModuleType("vaex.array_types")
    at.to_numpy = lambda x, strict=True: x

    class Encoding:
        def decode(self, typename, value, **kw):
            if typename == "_op":
                return ST.decode_op(value)
            if typename == "dtype":
                return types.SimpleNamespace(numpy=np.dtype(value))
            spec = dict(value)
            return types_[spec.pop("task-part-cpu-type")].decode(self, spec, **kw)
    vaex.cpu, vaex.array_types = cpu, at
    for name, mod in (("vaex", vaex), ("vaex.cpu", cpu), ("vaex.array_types", at)):
        monkeypatch.setitem(sys.modules, name, mod)
    replaced = vaex_plugin.install(legacy_statistic=True)
    assert set(replaced) == {"aggregations", "hash_map_unique_create", "legacy_statistic"}
    rng = np.random.default_rng(12)
    n = 100_000
    x, w1, w2 = rng.standard_normal(n), rng.standard_normal(n).astype("f4"), rng.standard_normal(n)
    sel = rng.random(n) < 0.4
    spec = {"task-part-cpu-type": "legacy_statistic", "expressions": ["x"], "shape": (12,), "selections": [None, "sel"],
            "op": {"code": 5, "reduce_function": "sum"}, "weights": ["w1", "w2"], "dtype": "float64", "minima": [-2.5], "maxima": [2.5],
            "edges": False, "selection_waslist": True}
    part = Encoding().decode("task-part-cpu", spec, df=None, nthreads=3)
    assert type(part).__name__ == "VaexTaskPartStatistic" and part.ideal_splits(8) == 1
    for t, i1 in enumerate(range(0, n, 30_000)):
        i2 = min(i1 + 30_000, n)
        part.process(t % 3, i1, i2, None, [None, sel[i1:i2]], [x[i1:i2], w1[i1:i2], w2[i1:i2]])
    part.reduce([])
    got = part.get_result()
    want = np.sum(np.array([SO.process([x], [w1, w2], [None, sel], SO.COV, [12], [-2.5], [2.5])]), axis=0)
    case = dict(binby=[x], weights=[w1, w2], selections=[None, sel], op=SO.COV, sizes=[12], minima=[-2.5], maxima=[2.5], edges=False)
    assert_grid(got, want, case)
    vaex_plugin.uninstall()
    assert types_["legacy_statistic"].__name__ == "TaskPartStatistic"


def test_reduce_semantics_nansum_against_sum():
    """MOMENTS reduce with nansum (a NaN sum becomes 0), COV with np.sum (a NaN product stays NaN)"""
    from vaex_b200 import statistic as ST, taskpart
    inf = np.array([np.inf, -np.inf, 1.0])
    p = taskpart.TaskPartStatistic(None, (), [], np.dtype("f8"), [None], ST.OP_ADD_WEIGHT_MOMENTS_01, ["a"], [], [], False, False)
    p.process(0, 0, 3, None, [None], [inf])
    assert np.array_equal(p.get_result(), [3.0, 0.0])
    p = taskpart.TaskPartStatistic(None, (), [], np.dtype("f8"), [None], ST.OP_COV, ["a", "b"], [], [], False, False)
    p.process(0, 0, 3, None, [None], [inf, np.ones(3)])
    r = p.get_result()
    assert np.isnan(r[2]) and r[0] == 3


def test_cov_1e8_rows_no_binby():
    import torch
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(0)
    cols = [torch.randn(n, device="cuda", generator=g, dtype=torch.float32) for _ in range(4)]
    from vaex_b200 import _lib, statistic as ST
    st = ST.Statistic(SO.COV, _lib.F32, [], [], [], False, 4, 1)
    st.bin(0, [], cols, [None], n, 0)
    got = st.read()[0]
    st.close()
    a = torch.stack(cols).double()
    s = a.sum(dim=1).cpu().numpy()
    prod = (a @ a.T).cpu().numpy()
    assert np.all(got[:4] == n)
    assert np.allclose(got[4:8], s, rtol=1e-9, atol=1e-6)
    assert np.all(got[8:24] == n)
    assert np.allclose(got[24:].reshape(4, 4), prod, rtol=1e-9, atol=1e-6)


if __name__ == "__main__":  # the profiling half of test_every_strategy_class_and_op, in a process of its own
    import json
    names = {}
    for strategy in STRATEGIES:
        for op in statistic_cases.OPS:
            for dtype in ("float32", "float64"):
                case = _strategy_case(strategy, op, dtype)
                names["%s-%d-%s" % (strategy, op, dtype)] = _kernels(lambda: device_grid(case, to_device=True))
    with open(sys.argv[1], "w") as f:
        json.dump(names, f)
