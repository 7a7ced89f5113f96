"""A numpy restatement of percentile_approx's finish (vaex/dataframe.py:1675-1780): the slicing of the count grid, the int64 cumulative
sum, the floor / ceil targets, the edge search and the interpolation, in the order and the types numpy evaluates the reference in.

The edge search is pluggable: `edges="numpy"` counts the cumulative entries below the target (left = max(c - 1, 0), right = min(c, P + 1));
`edges="vaexfast"` calls the compiled, unmodified vaexfast.grid_find_edges from oracle/_ref on the grid reshaped to (cells, P + 2), one
row per binby cell.  For 0 and 1 binby dimensions that is the reference's own call; for more it is what the reference's one-dimensional
code gives each cell (its multi-dimensional search reads outside the grid, DESIGN.md section 3)."""
import os

import numpy as np


def listify(x):
    """vaex.utils.listify for one argument"""
    if isinstance(x, str):
        return False, [x]
    try:
        x[0]
        return True, x
    except Exception:
        return False, [x]


def unlistify(waslist, x):
    return x if waslist else x[0]


def edges_numpy(cum, target):
    """-> (left, right) int64 arrays of the cells' shape"""
    plen = cum.shape[-1]
    c = np.sum(cum.astype(np.float64) < np.asarray(target)[..., None], axis=-1).astype(np.int64)
    return np.maximum(c - 1, 0), np.minimum(c, plen - 1)


def edges_vaexfast(cum, target):
    from oracle import ref_driver
    vf = ref_driver.vaexfast()
    plen = cum.shape[-1]
    cells = cum.shape[:-1]
    flat = np.ascontiguousarray(cum.reshape(-1, plen).astype(np.float64)) if cells else np.ascontiguousarray(cum.astype(np.float64))
    t = np.ascontiguousarray(np.asarray(target, np.float64).reshape(-1)) if cells else np.array(target, np.float64)
    out = np.zeros(flat.shape[:-1] + (2,), np.int64)
    vf.grid_find_edges(flat, t, out)
    return out[..., 0].reshape(cells), out[..., 1].reshape(cells)


def finish_one(counts, limit, percentage, edges="numpy"):
    """the reference's finish for one expression's count grid (binby axes first, the percentile axis last, edges included)"""
    find = edges_numpy if edges == "numpy" else edges_vaexfast
    nonnans = tuple([slice(2, -1)] * (counts.ndim - 1) + [slice(1, None)])
    c = counts[nonnans]
    cum = np.cumsum(c, -1)
    total = np.sum(c, -1)
    empty = total == 0
    plen = cum.shape[-1]
    waslist, percentages = listify(percentage)
    percentiles = []
    for p in percentages:
        if p == 0:
            percentiles.append(limit[0])
            continue
        if p == 100:
            percentiles.append(limit[1])
            continue
        values = np.array((total + 1) * p / 100.)
        values[empty] = 0
        floor_values = np.array(np.floor(values))
        ceil_values = np.array(np.ceil(values))

        def calculate_x(target):
            left, right = find(cum, target)
            left_value = np.take_along_axis(cum, np.asarray(left)[..., None], -1)[..., 0].astype(np.float64)
            right_value = np.take_along_axis(cum, np.asarray(right)[..., None], -1)[..., 0].astype(np.float64)
            denom = np.array(right_value - left_value)
            denom[denom == 0] = 1.0
            lb, ub = limit
            u = np.array(target - left_value) / denom
            xleft = lb + (np.asarray(left) - 0.5) * (ub - lb) / (plen - 3)
            xright = lb + (np.asarray(right) - 0.5) * (ub - lb) / (plen - 3)
            return xleft + (xright - xleft) * u

        x1 = calculate_x(floor_values)
        x2 = calculate_x(ceil_values)
        percentiles.append(x1 + (x2 - x1) * (values - floor_values))
    return unlistify(waslist, np.array(percentiles))


def percentile_approx(counts_list, limits, percentage, waslist, edges="numpy"):
    """finish over every expression, then finish2 (:1776-1779): np.array and unlistify over the expressions"""
    with np.errstate(all="ignore"):
        return unlistify(waslist, np.array([finish_one(c, lim, percentage, edges) for c, lim in zip(counts_list, limits)]))


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "percentile_golden.npz")


def load_golden():
    """tests/golden/percentile_golden.npz (tests/golden/make_golden_percentile.py): name -> dict(counts, limit, percentage, result,
    result_type), the limit and the percentage in the form the reference's finish was called with"""
    z = np.load(GOLDEN, allow_pickle=False)
    out = {}
    for name in sorted({k.split("/")[0] for k in z.files}):
        limit = z[name + "/limit"]
        if str(z[name + "/limit_kind"]) == "python":
            limit = [float(v) for v in limit]
        pct = z[name + "/pct"].tolist()
        out[name] = dict(counts=z[name + "/counts"], limit=limit, percentage=pct if bool(z[name + "/pct_list"]) else pct[0],
                         result=z[name + "/result"], result_type=str(z[name + "/result_type"]))
    return out


def limits_percentage(counts, vmin, vmax, percentage):
    """compute_limits of df.limits_percentage (vaex/dataframe.py:1825-1832) from the 16384-bin count between the minmax limits"""
    size = len(counts)
    cumcounts = np.concatenate([[0], np.cumsum(counts)])
    cumcounts = cumcounts / cumcounts.max()
    f = (1 - percentage / 100.) / 2
    x = np.linspace(vmin, vmax, size + 1)
    return np.interp([f, 1 - f], cumcounts, x)
