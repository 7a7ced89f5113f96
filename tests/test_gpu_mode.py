"""df.mode on the device: Frame.mode against the reference's own results (golden) and the numpy restatement, bit for bit, with host and
device columns, both count kernels, and the raising forms; Frame.skew / Frame.kurtosis against scipy."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import mode_oracle as MO  # noqa: E402
from helpers import same_bits, to_device  # noqa: E402

pytestmark = pytest.mark.gpu


def make_frame(cols, place, nthreads=3, filter=None):
    from vaex_b200 import execution, frame
    if place == "device":
        cols = {k: to_device(v) for k, v in cols.items()}
    ex = execution.Executor(nthreads, chunk_size=None if place == "device" else 700)
    return frame.Frame(cols, executor=ex, filter=filter)


def from_json(kwargs):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_mode import from_json as conv
    return conv(kwargs)


def case_columns(columns, kwargs, filt):
    names = set(kwargs["binby"]) | {kwargs["expression"]} | ({kwargs["selection"]} if kwargs.get("selection") else set())
    if filt:
        names.add(filt)
    return {k: columns[k] for k in names}


def device_ok(cols):
    """device columns carry no mask and only native byte order"""
    return not any(np.ma.isMaskedArray(v) or np.asarray(v).dtype.byteorder not in "=|<" for v in cols.values())


@pytest.mark.parametrize("place", ["host", "device"])
def test_golden(place):
    columns, cases = MO.load_golden()
    ran = 0
    for name, case in cases.items():
        kwargs = from_json(case["kwargs"])
        cols = case_columns(columns, kwargs, case["filter"])
        if place == "device" and not device_ok(cols):
            continue
        df = make_frame(cols, place, filter=case["filter"])
        kw = dict(kwargs)
        expression, binby = kw.pop("expression"), kw.pop("binby")
        if "error" in case:
            with pytest.raises(Exception) as info:
                df.mode(expression, binby, **kw)
            assert type(info.value).__name__ == case["error"], name
            continue
        got = df.mode(expression, binby, **kw)
        want = case["result"]
        assert got.shape == want.shape and got.dtype == want.dtype, (name, got.dtype, want.dtype)
        assert same_bits(got, want), name
        ran += 1
    assert ran >= (33 if place == "host" else 25)


@pytest.mark.parametrize("place", ["host", "device"])
def test_percentage_and_minmax_limits(place):
    rng = np.random.default_rng(11)
    n = 20000
    cols = dict(x=rng.normal(size=n), y=rng.normal(size=n).astype(np.float32), z=rng.random(n), s=rng.random(n) < 0.5)
    df = make_frame(cols, place)
    for kwargs in [dict(limits="90%", mode_limits="99%"), dict(limits="minmax", mode_limits=None), dict(limits=[[0, 1], "95%"])]:
        binby = ["z", "y"] if isinstance(kwargs["limits"], list) else ["y"]
        got = df.mode("x", binby, shape=16, mode_shape=16 if len(binby) == 2 else 32, selection="s", **kwargs)
        limits = [list(v) for v in df.limits(binby, kwargs["limits"])]
        mode_limits = list(df.limits(["x"], kwargs.get("mode_limits"))[0])
        want = MO.mode(cols, "x", binby, limits=limits, shape=16, mode_shape=16 if len(binby) == 2 else 32, mode_limits=mode_limits,
                       selection="s")
        assert same_bits(got, want), kwargs


def test_default_grids_and_mixed_placement():
    """mode's default 64 x 256 and 64 x 256^2 grids, a virtual expression, and a frame with host and device columns"""
    rng = np.random.default_rng(5)
    n = 300000
    cols = dict(x=rng.normal(size=n).astype(np.float32), y=rng.normal(size=n).astype(np.float32), v=rng.normal(size=n))
    from vaex_b200 import execution, frame
    df = frame.Frame(dict(x=to_device(cols["x"]), y=cols["y"], v=to_device(cols["v"])), executor=execution.Executor(2, chunk_size=65536))
    lim = [[-3, 3], [-3, 3]]
    got1 = df.mode("v", ["x"], limits=lim[:1], mode_limits=[-4, 4])
    assert same_bits(got1, MO.mode(cols, "v", ["x"], limits=lim[:1], mode_limits=[-4, 4]))
    got2 = df.mode("v + x", ["x", "y"], limits=lim, mode_limits=[-4, 4])
    cols2 = dict(cols, w=cols["v"] + cols["x"].astype(np.float64))
    assert got2.shape == (256, 256)
    assert same_bits(got2, MO.mode(cols2, "w", ["x", "y"], limits=lim, mode_limits=[-4, 4]))


def test_count_kernel_follows_the_grid_size():
    """the shared-memory count for grids whose 32-bit counts fit 96 KB, the global one above; kernel names recorded in a fresh
    process (torch.profiler loses device records late in a long one)"""
    script = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, %r)
from vaex_b200 import frame, execution
rng = np.random.default_rng(1)
n = 100000
df = frame.Frame(dict(x=torch.from_numpy(rng.normal(size=n)).cuda(), z=torch.from_numpy(rng.random(n)).cuda()), executor=execution.Executor(1))
out = {}
for label, shape, mode_shape in [("smem_2d", 300, 80), ("global_2d", 1000, 64), ("smem_3d", [20, 30], 40), ("global_3d", [40, 50], 64)]:
    binby = ["z"] if label.endswith("2d") else ["z", "x"]
    df.mode("x", binby, limits=[[0, 1], [-3, 3]][:len(binby)], shape=shape, mode_shape=mode_shape, mode_limits=[-3, 3])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        df.mode("x", binby, limits=[[0, 1], [-3, 3]][:len(binby)], shape=shape, mode_shape=mode_shape, mode_limits=[-3, 3])
        torch.cuda.synchronize()
    out[label] = sorted({e.name for e in prof.events() if "k_stat" in e.name})
print(json.dumps(out))
""" % ROOT
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    for label, kernels in names.items():
        count = [k for k in kernels if "k_stat_count_smem" in k or "k_stat_global" in k]
        assert len(count) == 1, (label, kernels)
        assert ("k_stat_count_smem" in count[0]) == label.startswith("smem"), (label, kernels)
        assert any("k_stat_mode" in k for k in kernels), (label, kernels)


def test_raises():
    rng = np.random.default_rng(2)
    cols = dict(a=rng.random(100), b=rng.random(100), c=rng.random(100), x=rng.normal(size=100))
    df = make_frame(cols, "host")
    with pytest.raises(ValueError, match="only supported with binby"):
        df.mode("x", [])
    with pytest.raises(IndexError):
        df.mode("x", ["a"], limits=[0, 1], mode_shape=1)
    with pytest.raises(ValueError, match="mode_shape equal to every binby size"):
        df.mode("x", ["a", "b", "c"], limits=[0, 1], shape=4, mode_shape=8)
    with pytest.raises(ValueError, match="mode_shape equal to every binby size"):
        df.mode("x", ["a", "b", "c"], limits=[0, 1], shape=[4, 4, 5], mode_shape=4)
    from vaex_b200 import _lib
    before = _lib.context().mem_stats()["live"]
    with pytest.raises(MemoryError, match="exceeds"):
        df.mode("x", ["a", "b"], limits=[0, 1], shape=[1 << 14, 1 << 14], mode_shape=64, mode_limits=[-3, 3])
    assert _lib.context().mem_stats()["live"] == before
    # the library refuses unequal sizes above three dimensions on its own
    from vaex_b200 import mode as _mode
    with pytest.raises(RuntimeError, match="equal sizes"):
        _mode.Histogram((4, 4, 4, 5), [0] * 4, [1] * 4)


@pytest.mark.parametrize("place", ["host", "device"])
def test_skew_kurtosis(place):
    from scipy import stats
    rng = np.random.default_rng(3)
    n = 50000
    x = rng.gamma(2.0, size=n)
    k = rng.integers(0, 8, n) + 0.5
    i = rng.integers(-50, 50, n).astype(np.int32)
    df = make_frame(dict(x=x, k=k, i=i), place)
    for name in ("x", "i"):
        v = (x if name == "x" else i).astype(np.float64)
        got_s, got_k = df.skew(name), df.kurtosis(name)
        want_s, want_k = stats.skew(v, bias=True), stats.kurtosis(v, bias=True)
        assert abs(got_s - want_s) <= 1e-12 * abs(want_s) and abs(got_k - want_k) <= 1e-12 * abs(want_k), name
        bs = df.skew(name, binby="k", limits=[0, 8], shape=8)
        bk = df.kurtosis(name, binby="k", limits=[0, 8], shape=8)
        for b in range(8):
            sel = v[k == b + 0.5]
            assert abs(bs[b] - stats.skew(sel, bias=True)) <= 1e-12 * abs(stats.skew(sel, bias=True)), (name, b)
            assert abs(bk[b] - stats.kurtosis(sel, bias=True)) <= 1e-12 * abs(stats.kurtosis(sel, bias=True)), (name, b)
