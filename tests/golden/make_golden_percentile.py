"""Generate tests/golden/percentile_golden.npz: count grids with edges and what the reference's own percentile_approx finish returns
for them.

    python tests/golden/make_golden_percentile.py [out.npz] [path/to/vaex/dataframe.py]

The `finish` closure of DataFrame.percentile_approx is taken from the reference's dataframe.py when this runs (ast, decorators
stripped) and executed with the compiled, unmodified vaexfast from oracle/_ref, vaex.utils' listify / unlistify, and the closure's free
variable `percentage` supplied as a global; finish2's `unlistify(waslist, np.array(results))` follows.  Only the inputs and the outputs
are stored.  Fixed zip timestamps make a rerun reproduce the archive byte for byte.

Per case `<name>/`: `counts` (int64, binby axes first, percentile axis last, edges included), `limit` (the limits pair, in `limit_kind`:
'array' = a numpy array as minmax returns it, 'python' = a list of Python floats), `pct` (percentages; int64 = Python ints) and
`pct_list` (a list, or one value), `result` and `result_type` (the type name of the returned object)."""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_edges import save  # noqa: E402

REFERENCE = "/root/reference/packages/vaex-core/vaex/dataframe.py"


def reference_finish(path):
    """the source of percentile_approx's nested `finish`, decorators stripped"""
    tree = ast.parse(open(path).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name == "percentile_approx":
            for inner in node.body:
                if isinstance(inner, ast.FunctionDef) and inner.name == "finish":
                    inner.decorator_list = []
                    return ast.unparse(inner)
    raise RuntimeError("percentile_approx's finish not found in " + path)


def listify(*args):
    if isinstance(args[0], str):
        return False, [[x] for x in args]
    try:
        _ = args[0][0]
        return True, args
    except Exception:
        return False, [[x] for x in args]


def unlistify(waslist, *args):
    if waslist:
        if len(args) == 1:
            return args[0]
        return args
    values = [x[0] for x in args]
    if len(values) == 1:
        return values[0]


def run_reference(source, counts, limit, percentage, waslist=False):
    from oracle import ref_driver
    vaex = types.SimpleNamespace(vaexfast=ref_driver.vaexfast(), utils=types.SimpleNamespace(listify=listify, unlistify=unlistify))
    scope = {"np": np, "vaex": vaex, "percentage": percentage}
    exec(source, scope)
    with np.errstate(all="ignore"):
        results = scope["finish"]([limit], [counts])
        return unlistify(waslist, np.array(results))


def grid(rng, binby, P, high=5, zero=0.3):
    shape = tuple(n + 3 for n in binby) + (P + 3,)
    g = rng.integers(0, high, shape).astype(np.int64)
    g[rng.random(shape) < zero] = 0
    return g


def cases():
    rng = np.random.default_rng(1632)
    out = {}

    def add(name, counts, limit, kind, pct, pct_list):
        out[name] = dict(counts=counts, limit=limit, kind=kind, pct=pct, pct_list=pct_list)

    f32 = np.array([-2.5, 3.25], np.float32)
    i64 = np.array([-7, 120], np.int64)
    py = [-4.0, 4.0]
    # no binby: int and float percentages, 0 and 100 mixed in
    for kind, lim in (("array", f32), ("array", i64), ("python", py)):
        tag = "python" if kind == "python" else lim.dtype.name
        add(f"nobinby_{tag}_int", grid(rng, [], 64), lim, kind, [0, 10, 25, 50, 99, 100], True)
        add(f"nobinby_{tag}_float", grid(rng, [], 64), lim, kind, [0.0, 12.5, 50.0, 77.7, 100.0], True)
        add(f"nobinby_{tag}_single", grid(rng, [], 33), lim, kind, [50], False)
    add("nobinby_single_zero", grid(rng, [], 16), f32, "array", [0], False)
    add("nobinby_single_hundred", grid(rng, [], 16), py, "python", [100.0], False)
    add("nobinby_empty", np.zeros(20, np.int64), py, "python", [25, 50.0], True)
    out_of_range = np.zeros(40, np.int64)
    out_of_range[[0, 1, 39]] = [5, 7, 11]  # NaN, underflow and overflow cells only
    add("nobinby_out_of_range", out_of_range, f32, "array", [10, 50, 90.0], True)
    add("nobinby_P1", grid(rng, [], 1), py, "python", [30, 50.0], True)
    add("nobinby_P1_f32", grid(rng, [], 1), f32, "array", [50], False)
    # 1-D binby: empty cells, ties (zero rows), int and float percentages
    for kind, lim in (("array", f32), ("array", i64), ("python", py)):
        tag = "python" if kind == "python" else lim.dtype.name
        add(f"binby1_{tag}_int", grid(rng, [9], 50, zero=0.6), lim, kind, [5, 50, 95], True)
        add(f"binby1_{tag}_float", grid(rng, [9], 50, zero=0.6), lim, kind, [33.3, 66.6], True)
        add(f"binby1_{tag}_single", grid(rng, [12], 20), lim, kind, [50], False)
    empty_cells = grid(rng, [7], 30)
    empty_cells[[2, 4, 5]] = 0
    add("binby1_empty_cells", empty_cells, py, "python", [25, 50, 75], True)
    out_of_range = np.zeros((8, 7), np.int64)
    out_of_range[[0, 1, 7], :] = 3  # rows outside the binby limits: every sliced cell stays empty ...
    out_of_range[3, [0, 1, 6]] = 4  # ... but one, whose rows all lie outside the percentile limits
    add("binby1_out_of_range", out_of_range, f32, "array", [50], False)
    add("binby1_P1", grid(rng, [6], 1), f32, "array", [20, 50.5], True)
    # totals above 2^53: an integer percentage multiplies in int64, a float one in double; the cumulative sums round to double
    big = grid(rng, [4], 24)
    big[2:-1, 3:10] = rng.integers(2**55, 2**57, (4, 7))
    add("binby1_big_int", big, py, "python", [50, 33], True)
    add("binby1_big_float", big, py, "python", [50.0, 33.0], True)
    add("nobinby_big_int", big[3], f32, "array", [50, 1, 99], True)
    add("nobinby_big_float", big[3], f32, "array", [50.0, 1.0, 99.0], True)
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "percentile_golden.npz")
    source = reference_finish(sys.argv[2] if len(sys.argv) > 2 else REFERENCE)
    arrays = {}
    for name, c in cases().items():
        limit = c["limit"] if c["kind"] == "array" else [float(v) for v in c["limit"]]
        pct = c["pct"] if c["pct_list"] else c["pct"][0]
        result = run_reference(source, c["counts"], limit, pct)
        arrays[name + "/counts"] = c["counts"]
        arrays[name + "/limit"] = np.asarray(c["limit"])
        arrays[name + "/limit_kind"] = np.array(c["kind"])
        arrays[name + "/pct"] = np.array(c["pct"])
        arrays[name + "/pct_list"] = np.array(c["pct_list"])
        arrays[name + "/result"] = np.asarray(result)
        arrays[name + "/result_type"] = np.array(type(result).__name__)
    save(path, arrays)
    print("wrote", len(arrays) // 7, "cases,", os.path.getsize(path) // 1024, "KiB")
