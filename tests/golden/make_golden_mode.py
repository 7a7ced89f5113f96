"""Generate tests/golden/mode_golden.npz: columns, df.mode calls on them and what the reference's own method returns.

    python tests/golden/make_golden_mode.py [out.npz] [path/to/vaex-core/vaex]

DataFrame.mode is taken from the reference's dataframe.py when this runs (ast, decorators stripped) and `legacy._asfloat` from
legacy.py.  It runs against a stub `self`: `limits` passes explicit pairs through and computes "minmax" with the compiled vaexfast
(oracle/ref_driver.minmax), `self(*expressions)` returns a subspace whose `histogram` is TaskHistogram.map (vaex/legacy.py:56-101)
over the compiled, unmodified vaexfast histogram2d / histogram3d / histogramNd in 1M-row chunks, and `selected()` keeps the rows of
the case's selection column.  Blocks are made native before `_asfloat`, as the reference's evaluation hands them over.

Where the reference writes outside its grid (a 3-D bin that rounds up to the size, an infinite minimum) or the restatement raises on
purpose (three binby of unequal sizes), the case holds the restatement's answer (tests/mode_oracle.py) and `reference` is false.
Only inputs and outputs are stored.  Fixed zip timestamps make a rerun reproduce the archive byte for byte."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from make_golden_edges import save  # noqa: E402
from make_golden_mutual_information import functions  # noqa: E402

import mode_oracle as MO  # noqa: E402

REFERENCE = "/root/reference/packages/vaex-core/vaex"


def reference_method(vaex_dir):
    scope = {"np": np}
    exec(functions(os.path.join(vaex_dir, "legacy.py"), ["_asfloat"]), scope)
    exec(functions(os.path.join(vaex_dir, "dataframe.py"), ["mode"], cls="DataFrame"), scope)
    return scope["mode"], scope["_asfloat"]


def native(a):
    if np.ma.isMaskedArray(a):
        return np.ma.array(np.ma.getdata(a).astype(a.dtype.newbyteorder("=")), mask=np.ma.getmaskarray(a))
    return np.asarray(a).astype(a.dtype.newbyteorder("="))


class Subspace:
    def __init__(self, stub, expressions, masked=False):
        self.stub, self.expressions, self.masked = stub, expressions, masked

    def selected(self):
        return Subspace(self.stub, self.expressions, True)

    def histogram(self, limits, size, progressbar=False, chunk=1024 * 1024):
        from oracle import ref_driver
        vf = ref_driver.vaexfast()
        data = np.zeros(size, np.float64)
        ranges_flat = [float(v) for lim in limits for v in lim]
        minima, maxima = [float(lim[0]) for lim in limits], [float(lim[1]) for lim in limits]
        columns = [native(self.stub.columns[e]) for e in self.expressions]
        n = len(columns[0])
        for i1 in range(0, n, chunk):
            blocks = [self.stub.asfloat(c[i1:i1 + chunk]) for c in columns]
            if self.masked:
                keep = np.asarray(self.stub.columns[self.stub.selection][i1:i1 + chunk], bool)
                blocks = [b[keep] for b in blocks]
            blocks = [np.ascontiguousarray(np.ma.getdata(b)) for b in blocks]
            if len(blocks) == 2:
                vf.histogram2d(blocks[0], blocks[1], None, data, *ranges_flat)
            elif len(blocks) == 3:
                vf.histogram3d(blocks[0], blocks[1], blocks[2], None, data, *ranges_flat)
            else:
                vf.histogramNd(list(blocks), None, data, minima, maxima)
        return data


class Stub:
    """the `self` the reference's method calls"""

    def __init__(self, columns, asfloat, selection=None):
        self.columns, self.asfloat, self.selection = columns, asfloat, selection

    def __call__(self, *expressions):
        return Subspace(self, list(expressions))

    def limits(self, expressions, value=None):
        """df.limits for explicit pairs and "minmax" / None, one value for all expressions or one per expression"""
        from oracle import ref_driver
        if value is None or isinstance(value, str) or np.isscalar(value[0]):
            value = [value] * len(expressions)
        return [ref_driver.minmax(self.columns[e]) if v is None or v == "minmax" else v for e, v in zip(expressions, value)]


def frame(rng, n=3000):
    x = rng.normal(size=n)
    x[::97] = np.nan
    x[5], x[6] = np.inf, -np.inf
    cols = dict(x=x, y=rng.normal(size=n).astype(np.float32), z=rng.random(n), w=rng.random(n), v=rng.random(n),
                a=rng.random(n), b=rng.random(n), c=rng.random(n))
    for dt in ("i1", "i2", "i4", "i8", "u1", "u2", "u4", "u8"):
        cols["n" + dt] = rng.integers(0, 40, n).astype(dt)
    cols["bool"] = rng.random(n) < 0.3
    cols["xb"] = rng.normal(size=n).astype(">f8")
    cols["yb"] = rng.normal(size=n).astype(">f4")
    cols["ib"] = rng.integers(-20, 20, n).astype(">i4")
    raw = rng.normal(size=n)
    raw[rng.random(n) < 0.2] = 50.0  # masked rows hold 50: vaexfast counts them there
    cols["m"] = np.ma.array(raw, mask=raw == 50.0)
    cols["s"] = rng.random(n) < 0.4
    cols["flt"] = x > -0.5
    # the value edges of limits [-1, 1] and [0, 1]: at min, at max, just below max, NaN, +-inf
    below = np.nextafter(1.0, 0.0)
    e = np.array([-1.0, 1.0, below, 0.0, np.nan, np.inf, -np.inf, -1.0, below, below])
    cols["e"] = np.resize(e, n)
    cols["t"] = np.resize(np.array([0.1, 0.1, 0.6, 0.6, 0.3]), n)  # two bins tie in every cell
    cols["k"] = np.resize(np.array([0.1, 0.3, 0.6, 0.8]), n)
    return cols


CASES = [
    ("x_by_z", dict(expression="x", binby=["z"], limits=[0, 1], shape=16, mode_shape=32, mode_limits=[-3, 3])),
    ("defaults_nonfinite_limits", dict(expression="y", binby=["x"])),  # minmax of x is +-inf: histogram2d counts nothing
    ("defaults", dict(expression="y", binby=["z"])),
    ("smem_sized", dict(expression="x", binby=["z"], limits=[0, 1], shape=300, mode_shape=80, mode_limits=[-3, 3])),
    ("global_sized", dict(expression="x", binby=["z"], limits=[0, 1], shape=1000, mode_shape=64, mode_limits=[-3, 3])),
    ("nonfinite_mode_limits_2d", dict(expression="x", binby=["z"], limits=[0, 1], shape=8, mode_shape=8, mode_limits=[-np.inf, 3])),
    ("three_d_unequal", dict(expression="x", binby=["z", "y"], limits=[[0, 1], [-2, 2]], shape=[5, 7], mode_shape=9, mode_limits=[-3, 3])),
    ("three_d_minmax", dict(expression="z", binby=["y", "w"], shape=6, mode_shape=10)),
    ("three_d_global", dict(expression="x", binby=["z", "w"], limits=[0, 1], shape=[40, 50], mode_shape=64, mode_limits=[-3, 3])),
    ("four_d", dict(expression="z", binby=["a", "b", "c"], limits=[0, 1], shape=4, mode_shape=4, mode_limits=[0, 1])),
    ("selection", dict(expression="x", binby=["z"], limits=[0, 1], shape=12, mode_shape=20, mode_limits=[-3, 3], selection="s")),
    ("selection_3d", dict(expression="x", binby=["z", "w"], limits=[0, 1], shape=[3, 4], mode_shape=20, mode_limits=[-3, 3], selection="s")),
    ("masked", dict(expression="m", binby=["z"], limits=[0, 1], shape=6, mode_shape=16, mode_limits=[-3, 60])),
    ("masked_binby", dict(expression="z", binby=["m"], limits=[-3, 60], shape=6, mode_shape=8, mode_limits=[0, 1])),
    ("edges_2d", dict(expression="e", binby=["z"], limits=[0, 1], shape=3, mode_shape=64, mode_limits=[-1, 1])),
    ("edges_2d_binby", dict(expression="z", binby=["e"], limits=[-1, 1], shape=64, mode_shape=4, mode_limits=[0, 1])),
    ("edges_3d_in_bounds", dict(expression="e", binby=["z", "w"], limits=[0, 1], shape=2, mode_shape=64, mode_limits=[0, 1])),
    ("ties", dict(expression="t", binby=["k"], limits=[0, 1], shape=4, mode_shape=10, mode_limits=[0, 1])),
    ("empty_cells", dict(expression="z", binby=["k"], limits=[0, 1], shape=20, mode_shape=10, mode_limits=[0, 1])),
    ("empty_binby", dict(expression="x", binby=[])),
    ("mode_shape_1", dict(expression="x", binby=["z"], limits=[0, 1], shape=4, mode_shape=1, mode_limits=[-3, 3])),
] + [("dtype_" + dt, dict(expression="n" + dt, binby=["z"], limits=[0, 1], shape=5, mode_shape=16)) for dt in
     ("i1", "i2", "i4", "i8", "u1", "u2", "u4", "u8")] + [
    ("dtype_bool", dict(expression="bool", binby=["z"], limits=[0, 1], shape=5, mode_shape=4, mode_limits=[0, 2])),
    ("int_binby", dict(expression="z", binby=["ni4", "nu1"], shape=[6, 5], mode_shape=7, mode_limits=[0, 1])),
    ("byteswapped", dict(expression="xb", binby=["z"], limits=[0, 1], shape=7, mode_shape=12)),
    ("byteswapped_3d", dict(expression="yb", binby=["ib", "w"], limits=[[-20, 20], [0, 1]], shape=[5, 6], mode_shape=9)),
]

# where the reference writes outside its grid, or the restatement refuses on purpose: the restatement's answer
DEPARTURES = [
    ("edges_3d_round_up", dict(expression="e", binby=["z", "w"], limits=[0, 1], shape=2, mode_shape=64, mode_limits=[-1, 1])),
    ("edges_3d_binby_round_up", dict(expression="z", binby=["e", "w"], limits=[[-1, 1], [0, 1]], shape=[3, 64], mode_shape=4, mode_limits=[0, 1])),
    ("infinite_minimum_3d", dict(expression="x", binby=["z", "w"], limits=[0, 1], shape=2, mode_shape=8, mode_limits=[-np.inf, 3])),
    ("four_d_unequal", dict(expression="z", binby=["a", "b", "c"], limits=[0, 1], shape=4, mode_shape=8)),
]

FILTERED = [("filtered", dict(expression="x", binby=["z"], limits=[0, 1], shape=10, mode_shape=16, mode_limits=[-3, 3]), "flt"),
            ("filtered_3d", dict(expression="y", binby=["z", "w"], limits=[0, 1], shape=[4, 3], mode_shape=16, mode_limits=[-3, 3]), "flt")]


def jsonable(kwargs):
    def conv(v):
        if isinstance(v, (list, tuple)):
            return [conv(k) for k in v]
        if isinstance(v, float) and not np.isfinite(v):
            return repr(v)
        return v
    return {k: conv(v) for k, v in kwargs.items()}


def from_json(kwargs):
    """the stored keyword arguments, infinities restored"""
    def conv(v):
        if isinstance(v, list):
            return [conv(k) for k in v]
        if v in ("inf", "-inf"):
            return float(v)
        return v
    return {k: conv(v) for k, v in kwargs.items()}


def run_reference(method, asfloat, columns, kwargs):
    kw = dict(kwargs)
    stub = Stub(columns, asfloat, selection=kw.get("selection"))
    with np.errstate(all="ignore"):
        return method(stub, **kw)


def cases(vaex_dir=REFERENCE):
    method, asfloat = reference_method(vaex_dir)
    columns = frame(np.random.default_rng(2006))
    arrays = {"columns": json.dumps(sorted(columns))}
    for k, v in columns.items():
        arrays["col_" + k] = np.ma.getdata(v)
        if np.ma.isMaskedArray(v):
            arrays["mask_" + k] = np.ma.getmaskarray(v)
    names = []

    def store(name, kwargs, filt, reference, fn):
        meta = {"kwargs": jsonable(kwargs), "filter": filt, "reference": reference}
        cols = columns if filt is None else {k: v[np.asarray(columns[filt], bool)] for k, v in columns.items()}
        try:
            result = fn(cols, kwargs)
            arrays["result_" + name] = np.asarray(result)
        except Exception as e:
            meta["error"] = type(e).__name__
        arrays["meta_" + name] = json.dumps(meta)
        names.append(name)

    for name, kwargs in CASES:
        store(name, kwargs, None, True, lambda c, kw: run_reference(method, asfloat, c, kw))
    for name, kwargs, filt in FILTERED:
        store(name, kwargs, filt, True, lambda c, kw: run_reference(method, asfloat, c, kw))
    for name, kwargs in DEPARTURES:
        store(name, kwargs, None, False, lambda c, kw: MO.mode(c, **kw))
    arrays["names"] = json.dumps(names)
    return arrays


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "mode_golden.npz")
    data = cases(sys.argv[2] if len(sys.argv) > 2 else REFERENCE)
    save(path, data)
    print("wrote", len(data), "arrays,", os.path.getsize(path) // 1024, "KiB")
