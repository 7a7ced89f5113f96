"""Generate tests/golden/mutual_information_golden.npz: columns, mutual_information calls on them and what the reference's own
method returns.

    python tests/golden/make_golden_mutual_information.py [out.npz] [path/to/vaex-core/vaex]

DataFrame.mutual_information is taken from the reference's dataframe.py when this runs (ast, the `docsubst` and `delayed` decorators
stripped), with kld.mutual_information and utils.disjoined / multisum / _issequence / _expand_shape from kld.py and utils.py the same
way.  It runs against a stub `self`: `count` returns grids of the compiled, unmodified superagg in oracle/_ref (sliced [2:-1] as
count(edges=False) does), `limits` returns minmax from the compiled vaexfast or passes explicit pairs through, and `_delay` is the
identity.  Only inputs and outputs are stored: per case its keyword arguments (JSON), the result, the result's type name, the sort
labels (JSON), or the type name of the exception it raised.  Fixed zip timestamps make a rerun reproduce the archive byte for byte.

Two frames: `local` holds the reference's df_local columns `x` .. `ints` (reference tests/common.py:313-381, `z` = x + t * y with
t = 1 stored as data); `rows` holds 3000 seeded rows `a`, `b`, `c`, `w` (float32 with NaN), `k` (int32) and `sel` (a boolean
selection).  The `df_local_*` cases run on the rows where the boolean column `flt` = (x >= 0) & (x < 10) holds, the reference's
filtered df_local (tests/common.py:308-311); their `filter` names it, and every case names its frame."""
import ast
import itertools
import json
import numbers
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_edges import save  # noqa: E402
from make_golden_percentile import listify, unlistify  # noqa: E402  (the vaex.utils stand-ins)

REFERENCE = "/root/reference/packages/vaex-core/vaex"


def functions(path, names, cls=None):
    """the sources of the named functions of a module (or of class `cls`), decorators stripped"""
    tree = ast.parse(open(path).read())
    body = tree.body
    if cls is not None:
        body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls).body
    out = []
    for node in body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            for inner in ast.walk(node):
                if isinstance(inner, ast.FunctionDef):
                    inner.decorator_list = []
            out.append(ast.unparse(node))
    if len(out) != len(names):
        raise RuntimeError(f"{names} not all found in {path}")
    return "\n\n".join(out)


def _is_limit(x):
    return isinstance(x, (tuple, list, np.ndarray)) and all(isinstance(k, numbers.Number) for k in x)


def reference_method(vaex_dir):
    scope = {"np": np, "itertools": itertools, "default_shape": 128, "delayed_list": lambda x: x}
    exec(functions(os.path.join(vaex_dir, "utils.py"), ["multisum", "disjoined", "_issequence", "_expand_shape"]), scope)
    utils = types.SimpleNamespace(listify=listify, unlistify=unlistify, disjoined=scope["disjoined"], multisum=scope["multisum"])
    kld_scope = {"np": np, "vaex": types.SimpleNamespace(utils=utils)}
    exec(functions(os.path.join(vaex_dir, "kld.py"), ["mutual_information"]), kld_scope)
    scope["vaex"] = types.SimpleNamespace(utils=utils, kld=types.SimpleNamespace(mutual_information=kld_scope["mutual_information"]))
    scope["_issequence"] = scope["_issequence"]
    exec(functions(os.path.join(vaex_dir, "dataframe.py"), ["mutual_information"], cls="DataFrame"), scope)
    return scope["mutual_information"]


class Stub:
    """the `self` the reference's method calls: count, limits and _delay over numpy columns"""

    def __init__(self, columns):
        self.columns = columns

    def _delay(self, delay, value):
        return value

    def _minmax(self, e):
        from oracle import ref_driver
        return ref_driver.minmax(self.columns[e])

    def _one(self, e, v):
        if _is_limit(v):
            return v
        if v is None or v == "minmax":
            return self._minmax(e)
        raise ValueError(v)

    def limits(self, expression, value=None, delay=False, selection=None):
        """df.limits (vaex/dataframe.py:1844-2004) for names, lists of names and lists of name tuples"""
        if expression == []:
            return []
        waslist, (expressions,) = listify(expression)
        if value is None:
            value = "minmax"
        values = (value,) * len(expressions) if _is_limit(value) or not isinstance(value, (tuple, list, np.ndarray)) else value
        out = []
        for e, v in zip(expressions, values):
            if isinstance(e, (tuple, list, np.ndarray)):
                inner = (v,) * len(e) if _is_limit(v) or not isinstance(v, (tuple, list, np.ndarray)) else v
                out.append([self._one(ee, vv) for ee, vv in zip(e, inner)])
            else:
                out.append(self._one(e, v))
        return unlistify(waslist, out)

    def count(self, binby, limits, shape, delay=False, selection=False):
        from oracle import ref_driver
        specs = []
        for e, (lo, hi), n in zip(binby, limits, shape):
            col = self.columns[e]
            data = np.ma.getdata(col) if np.ma.isMaskedArray(col) else np.asarray(col)
            mask = np.ma.getmaskarray(col) if np.ma.isMaskedArray(col) else None
            specs.append(dict(kind="scalar", data=data, mask=mask, vmin=float(lo), vmax=float(hi), bins=int(n)))
        sel = None if selection is None or selection is False else np.ascontiguousarray(self.columns[selection], bool)
        grid, = ref_driver.binby(specs, [dict(op="count", data=None, mask=sel)])
        return grid[tuple([slice(2, -1)] * len(binby))]


def df_local():
    x = np.arange(-2, 40, dtype=">f8").reshape((-1, 21)).T.copy()[:, 0]
    y = x ** 2
    ints = np.arange(-2, 19, dtype="i8")
    for off in (0, 10):
        ints[0 + off], ints[1 + off], ints[2 + off] = 2**62 + 1, -2**62 + 1, -2**62 - 1
    ma_value = 77777
    m = x.copy()
    m[-1 + 10 + 2] = ma_value
    m[-1 + 20] = ma_value
    m = np.ma.array(m, mask=m == ma_value)
    n = x.copy()
    n[-2 + 10] = np.nan
    n[-2 + 20] = np.nan
    nm = n.copy()
    nm[-1 + 10] = ma_value
    nm[-1 + 20] = ma_value
    nm = np.ma.array(nm, mask=nm == ma_value)
    mi = np.ma.array(m.data.astype(np.int64), mask=m.data == ma_value)
    return dict(x=x, y=y, z=x + 1.0 * y, m=m, n=n, nm=nm, mi=mi, ints=ints)


def random_columns():
    rng = np.random.default_rng(685)
    N = 3000
    a = rng.normal(size=N)
    b = a + 0.5 * rng.normal(size=N)
    c = rng.uniform(-2, 2, N)
    w = (b * c + 0.1 * rng.normal(size=N)).astype(np.float32)
    w[rng.random(N) < 0.05] = np.nan
    k = rng.integers(-3, 9, N).astype(np.int32)
    sel = rng.random(N) < 0.6
    return dict(a=a, b=b, c=c, w=w, k=k, sel=sel)


LOCAL = {"df_local_known", "df_local_binby1", "df_local_binby2", "df_local_binby3", "df_local_sort_pairs", "pair_xy", "pair_yx", "pair_xx",
         "matrix", "list_vs_one", "list_vs_list", "pairs", "matrix_dim3", "nan_masked_matrix", "masked_int_pair"}


def cases(local):
    from oracle import ref_driver
    lx, ly = (ref_driver.minmax(local[e][local["flt"]]).tolist() for e in ("x", "y"))
    out = {}
    # reference tests/agg_test.py:443-463
    out["df_local_known"] = dict(x="x", y="y", mi_limits=[lx, ly], mi_shape=32)
    out["df_local_binby1"] = dict(x="x", y="y", mi_limits=[lx, ly], mi_shape=32, binby="x", limits=[0, 10], shape=2)
    out["df_local_binby2"] = dict(x="x", y="y", mi_limits=[lx, ly], mi_shape=32, binby=["x", "y"], limits=[[0, 10], [0, 100]], shape=[2, 3])
    out["df_local_binby3"] = dict(x="x", y="y", mi_limits=[lx, ly], mi_shape=32, binby=["x", "y", "z"], limits=[[0, 10], [0, 100], [-100, 100]],
                                  shape=[2, 3, 4])
    out["df_local_sort_pairs"] = dict(x=[["x", "y"], ["x", "z"]], sort=True)
    # reference tests/mutual_information_test.py, on df_local
    out["pair_xy"] = dict(x="x", y="y")
    out["pair_yx"] = dict(x="y", y="x")
    out["pair_xx"] = dict(x="x", y="x")
    out["matrix"] = dict(x=["x", "y", "z"])
    out["list_vs_one"] = dict(x=["x", "y", "z"], y="z")
    out["list_vs_list"] = dict(x=["x", "y", "z"], y=["y", "z"])
    out["pairs"] = dict(x=[["x", "y"], ["x", "z"], ["y", "z"]])
    out["matrix_dim3"] = dict(x=["x", "y"], dimension=3, mi_shape=4)
    # NaN and masked values
    out["nan_masked_matrix"] = dict(x=["n", "nm", "m", "mi"], mi_shape=8)
    out["masked_int_pair"] = dict(x="mi", y="ints", mi_shape=5)
    # seeded rows: binby of 0-3 dimensions, mi_shape per axis, 1 and 2, float32 with NaN, int32, selections, empty cells
    out["ab_256"] = dict(x="a", y="b")
    out["ab_shapes"] = dict(x="a", y="b", mi_shape=[7, 3])
    out["ab_shape1"] = dict(x="a", y="b", mi_shape=1)
    out["ab_shape2"] = dict(x="a", y="b", mi_shape=2)
    out["ab_dimension1"] = dict(x=["a", "b"], dimension=1, mi_shape=16)
    out["abc_dim3"] = dict(x=["a", "b", "c"], dimension=3, mi_shape=5)
    out["wk_pair"] = dict(x="w", y="k", mi_shape=[9, 12])
    out["ab_binby1"] = dict(x="a", y="b", mi_shape=16, binby=["c"], shape=5)
    out["ab_binby2"] = dict(x="a", y="b", mi_shape=[6, 10], binby=["c", "k"], shape=[3, 4], limits=[[-2, 2], [-3, 9]])
    out["ab_binby3"] = dict(x="a", y="b", mi_shape=4, binby=["c", "k", "w"], shape=[2, 3, 2])
    out["pairs_binby1"] = dict(x=[["a", "b"], ["b", "c"], ["a", "c"]], mi_shape=8, binby=["k"], shape=4)
    out["matrix_binby1"] = dict(x=["a", "b"], mi_shape=8, binby=["c"], shape=3)
    out["list_vs_list_binby2"] = dict(x=["a", "b"], y=["c", "w"], mi_shape=6, binby=["k", "c"], shape=[2, 3])
    out["empty_cells"] = dict(x="a", y="b", mi_shape=8, binby=["c"], limits=[-3, 3], shape=6)
    out["all_empty"] = dict(x="a", y="b", mi_shape=8, mi_limits=[100, 200])
    out["selection"] = dict(x=["a", "b", "c"], mi_shape=16, selection="sel")
    out["selection_binby1"] = dict(x="a", y="w", mi_shape=10, binby=["c"], shape=3, selection="sel")
    # mi_limits go to the sorted, deduplicated combinations
    out["mi_limits_sorted"] = dict(x=[["b", "a"], ["c", "a"]], mi_limits=[[[-1, 1], [-3, 3]], [[-0.5, 0.5], [-2, 2]]], mi_shape=12)
    out["mi_limits_pair_per_axis"] = dict(x="b", y="a", mi_limits=[[-1, 1], [-3, 3]], mi_shape=12)
    out["mi_limits_one_pair"] = dict(x=["a", "b", "c"], mi_limits=[-1.5, 1.5], mi_shape=12)
    # the sort quirks
    out["sort_single_pair"] = dict(x="ab", y="b", sort=True, mi_shape=8)
    out["sort_list_vs_one"] = dict(x=["c", "a", "b"], y="a", sort=True, mi_shape=8)
    out["sort_matrix_index_error"] = dict(x=["a", "b", "c"], sort=True, mi_shape=8)
    out["sort_binby_raises"] = dict(x=[["a", "b"], ["a", "c"]], sort=True, mi_shape=8, binby=["k"], shape=3)
    # raising forms
    out["binby_dim4"] = dict(x="a", y="b", mi_shape=2, binby=["a", "b", "c", "k"], shape=2)
    out["string_x_list_y"] = dict(x="ab", y=["a", "b"], mi_shape=4)
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "mutual_information_golden.npz")
    method = reference_method(sys.argv[2] if len(sys.argv) > 2 else REFERENCE)
    local = df_local()
    local["flt"] = (local["x"] >= 0) & (local["x"] < 10)  # df_local is the filtered frame of reference tests/common.py:308-311
    rows = random_columns()
    rows["ab"] = rows["a"]  # a two-character name for the single-string sort and x-string forms
    frames = dict(local=local, rows=rows)
    arrays = {}
    for frame, columns in frames.items():
        for name, col in columns.items():
            key = "frames/" + frame + "/" + name
            arrays[key] = np.ma.getdata(col) if np.ma.isMaskedArray(col) else col
            if np.ma.isMaskedArray(col):
                arrays[key + "/mask"] = np.ma.getmaskarray(col)
    for name, kwargs in cases(local).items():
        p = "cases/" + name + "/"
        arrays[p + "kwargs"] = np.array(json.dumps(kwargs, sort_keys=True))
        frame = "local" if name in LOCAL else "rows"
        flt = "flt" if name.startswith("df_local") else ""
        arrays[p + "frame"] = np.array(frame)
        arrays[p + "filter"] = np.array(flt)
        columns = frames[frame]
        on = Stub({k: v[columns[flt]] for k, v in columns.items()} if flt else columns)
        try:
            with np.errstate(all="ignore"):
                result = method(on, **kwargs)
        except Exception as e:  # the raising forms keep the exception's type
            arrays[p + "error"] = np.array(type(e).__name__)
            arrays[p + "result_type"] = np.array("exception")
            continue
        arrays[p + "result_type"] = np.array(type(result).__name__)
        if isinstance(result, tuple):
            values, labels = result
            arrays[p + "result"] = np.asarray(values)
            arrays[p + "labels"] = np.array(json.dumps([list(v) if isinstance(v, tuple) else v for v in labels]))
        else:
            arrays[p + "result"] = np.asarray(result)
    save(path, arrays)
    print("wrote", len(cases(local)), "cases,", os.path.getsize(path) // 1024, "KiB")
