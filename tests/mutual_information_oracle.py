"""A numpy restatement of df.mutual_information (vaex/dataframe.py:685-819): the argument forms, the sorted and deduplicated
combinations, the count grids (from the C oracle's count path, oracle/binstats_oracle.c), the per-cell kld.mutual_information
(vaex/kld.py:13-21) with the marginals of vaex.utils.disjoined / multisum (vaex/utils.py:172-195) and the assembly of the result,
in float64 and in numpy's order.  It also states the per-cell bound that the device finish holds against it (DESIGN.md section 3)."""
import itertools
import os

import numpy as np

U = 2.0 ** -53


def seq(v):
    return isinstance(v, (tuple, list, np.ndarray))


def forms(x, y=None, dimension=2, mi_limits=None):
    """-> (combinations, result shape, waslist, mi_limits) for the five ways of asking"""
    if y is None and seq(x) and len(x) and all(seq(k) for k in x):
        return x, (len(x),), True, mi_limits
    if seq(x) and y is None:
        return list(itertools.product(x, repeat=dimension)), (len(x),) * dimension, True, mi_limits
    if seq(x) and seq(y):
        pairs = [[str(i), str(j)] for j in x for i in y]  # np.array(...).tolist() of the reference makes every name a str
        return pairs, (len(x), len(y)), True, mi_limits
    if seq(x):
        return [(i, y) for i in x], (len(x),), True, mi_limits
    if seq(y):
        return [(i, y) for i in x], (len(y),), True, mi_limits
    return [(x, y)], (), False, ([mi_limits] if mi_limits else mi_limits)


def dedupe(combinations):
    keys = [tuple(sorted(c)) for c in combinations]
    unique, inverse = np.unique(keys, return_inverse=True, axis=0)
    return [tuple(u) for u in unique.tolist()], inverse


def marginals(counts):
    """disjoined's one-dimensional sums: axis k keeps only itself, the others summed with nansum from the first axis on"""
    out = []
    for k in range(counts.ndim):
        m = counts
        for removed, axis in enumerate(a for a in range(counts.ndim) if a != k):
            m = np.nansum(m, axis=axis - removed)
        out.append(m)
    return out


def product_of_marginals(counts):
    q = None
    for k, m in enumerate(marginals(counts)):
        shape = [1] * counts.ndim
        shape[k] = len(m)
        q = m.reshape(shape) if q is None else q * m.reshape(shape)
    return q


def mi_cell(counts):
    """kld.mutual_information of one float64 grid: 0.0 when it is empty (P = 0/0 leaves the mask empty)"""
    with np.errstate(invalid="ignore", divide="ignore"):
        P = counts / counts.sum()
        Q = product_of_marginals(counts)
        Q = Q / Q.sum()
        keep = (P > 0) & (Q > 0)
        return np.sum(P[keep] * np.log(P[keep] / Q[keep]))


def calculate(counts, nbinby, per_cell=None):
    """`calculate` (:766-790): the counts as float64, then mi_cell of every binby cell (the binby axes last); with `per_cell`
    (e.g. `bound`) that function of every cell's int64 counts instead"""
    if per_cell is None:
        counts, per_cell = counts.astype(np.float64), mi_cell
    if nbinby > 3:
        raise ValueError("binby with dim > 3 is not yet supported")
    if nbinby == 0:
        return per_cell(counts)
    cells = counts.shape[counts.ndim - nbinby:]
    out = np.zeros(cells, dtype=float)
    for index in np.ndindex(*cells):
        out[index] = per_cell(counts[(Ellipsis,) + index])
    return out


def bound(counts):
    """|device − reference| for one cell's grid (int64 counts, no edges), DESIGN.md section 3: with u = 2^-53, d MI axes,
    n = the cells of the grid, h = ceil(log2 n) + ceil(n / 256) + 40 (the longest chain of additions a term passes through, on the
    device or in numpy's pairwise sum) and S = Σ_{c > 0} P·(|log P| + |log Q|),
        (3d + 4)·(h + 2)·u + (3h + 24)·u·S"""
    c = counts.astype(np.float64)
    N = c.sum()
    if N == 0:
        return 0.0
    d = counts.ndim
    P = c / N
    Q = product_of_marginals(c) / N ** d
    keep = P > 0
    S = np.sum(P[keep] * (np.abs(np.log(P[keep])) + np.abs(np.log(Q[keep]))))
    n = c.size
    h = int(np.ceil(np.log2(max(n, 2)))) + -(-n // 256) + 40
    return (3 * d + 4) * (h + 2) * U + (3 * h + 24) * U * S


def assemble(mi_list, x, inverse, binby_shape, shape_result, waslist, sort):
    mi = np.array(mi_list)
    if sort:
        order = np.argsort(mi)[::-1]
        labels = [x[k] for k in order]  # before mi[order]: with binby this is what raises
        return mi[order], labels
    mi = mi[inverse]
    return np.array(mi if waslist else mi[0]).reshape(tuple(binby_shape) + tuple(shape_result))


def count_grid(columns, expressions, limits, shapes, selection=None):
    """count(binby=expressions, limits, shape, edges=False) through the C oracle: the grid sliced [2:-1] on every axis"""
    from oracle import oracle as O
    specs = []
    for e, (lo, hi), n in zip(expressions, limits, shapes):
        col = columns[e]
        data = np.ma.getdata(col) if np.ma.isMaskedArray(col) else np.asarray(col)
        mask = np.ma.getmaskarray(col) if np.ma.isMaskedArray(col) else None
        specs.append(O.scalar(data, lo, hi, n, mask=mask))
    sel = None if selection is None else np.asarray(columns[selection], bool)
    grid, = O.binby(specs, [O.agg("count", mask=sel)])
    return grid[tuple([slice(2, -1)] * len(expressions))]


def minmax(column):
    col = column
    if np.ma.isMaskedArray(col):
        col = np.asarray(col.data)[~np.ma.getmaskarray(col)]
    col = np.asarray(col)
    col = col.astype(col.dtype.newbyteorder("="))
    if col.dtype.kind == "f":
        col = col[~np.isnan(col)]
    return np.array([col.min(), col.max()], col.dtype)


def limits_of(columns, expressions, value):
    """df.limits for a flat list of names: "minmax" / None per name, or explicit pairs passed through"""
    values = (value,) * len(expressions) if (value is None or isinstance(value, str) or all(not seq(v) for v in value)) else value
    return [minmax(columns[e]) if (v is None or v == "minmax") else v for e, v in zip(expressions, values)]


def mutual_information(columns, x, y=None, dimension=2, mi_limits=None, mi_shape=256, binby=(), limits=None, shape=128, sort=False,
                       selection=None, per_cell=None):
    """the whole method over a dict of numpy columns; a string binby is one expression.  per_cell=bound gives every value's bound
    in the layout of the result"""
    combinations, shape_result, waslist, mi_limits = forms(x, y, dimension, mi_limits)
    binby = [binby] if isinstance(binby, str) else list(binby)
    if len(binby) > 3:
        raise ValueError("binby with dim > 3 is not yet supported")
    binby_shape = tuple(shape) if seq(shape) else (shape,) * len(binby)
    binby_limits = limits_of(columns, binby, limits)
    unique, inverse = dedupe(combinations)
    per = (mi_limits,) * len(unique) if (mi_limits is None or isinstance(mi_limits, str) or all(not seq(v) for v in mi_limits)) else mi_limits
    mi_list = []
    for c, v in zip(unique, per):
        lims = limits_of(columns, list(c), v)
        mshape = tuple(mi_shape) if seq(mi_shape) else (mi_shape,) * len(c)
        counts = count_grid(columns, list(c) + binby, lims + binby_limits, mshape + binby_shape, selection)
        mi_list.append(calculate(counts, len(binby), per_cell))
    return assemble(mi_list, x, inverse, binby_shape, shape_result, waslist, sort)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mutual_information_golden.npz")


def load_golden():
    """tests/golden/mutual_information_golden.npz (tests/golden/make_golden_mutual_information.py): the frames (name -> columns),
    and per case its keyword arguments, its frame, the filter column (or None), the result (or the exception type name) and the result's type name"""
    import json
    z = np.load(GOLDEN, allow_pickle=False)
    frames = {}
    for k in z.files:
        if k.startswith("frames/") and not k.endswith("/mask"):
            _, frame, name = k.split("/")
            frames.setdefault(frame, {})[name] = np.ma.array(z[k], mask=z[k + "/mask"]) if k + "/mask" in z.files else z[k]
    cases = {}
    for name in sorted({k.split("/")[1] for k in z.files if k.startswith("cases/")}):
        p = "cases/" + name + "/"
        case = dict(kwargs=json.loads(str(z[p + "kwargs"])), result_type=str(z[p + "result_type"]), frame=str(z[p + "frame"]),
                    filter=str(z[p + "filter"]) or None)
        if p + "error" in z.files:
            case["error"] = str(z[p + "error"])
        else:
            case["result"] = z[p + "result"]
            if p + "labels" in z.files:
                case["labels"] = json.loads(str(z[p + "labels"]))
        cases[name] = case
    return frames, cases
