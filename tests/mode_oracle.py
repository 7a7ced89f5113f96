"""A numpy restatement of df.mode (vaex/dataframe.py:2006-2034) over vaex.legacy.TaskHistogram (vaex/legacy.py:22-110) and the
compiled vaexfast histogram2d / histogram3d / histogramNd (src/vaexfast.cpp:577-600, 818-860, 939-965), with the rules of DESIGN.md
section 3 where the reference writes outside its grid.

Columns are numpy arrays (masked arrays bin the values under their mask, as vaexfast reads them); `selection` and `filter` name
boolean columns whose rows are kept before binning."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mode_golden.npz")


def asfloat(a):
    """legacy._asfloat after the block was made native: every numeric dtype as float64, the values under a mask"""
    a = np.ma.getdata(a)
    return np.asarray(a).astype(a.dtype.newbyteorder("="), copy=False).astype(np.float64)


def minmax(a):
    """Frame.minmax / df.minmax: NaN and masked rows ignored, reduced in the compute class (float64 for float64 / int64, float32
    otherwise) and cast back to the column's dtype"""
    data = np.asarray(np.ma.getdata(a))
    dtype = data.dtype.newbyteorder("=")
    if np.ma.isMaskedArray(a):
        data = data[~np.ma.getmaskarray(a)]
    cls = np.float64 if dtype in (np.dtype("f8"), np.dtype("i8")) else np.float32
    v = data.astype(dtype).astype(cls)
    v = v[~np.isnan(v)]
    lo, hi = (v.min(), v.max()) if len(v) else (np.inf, -np.inf)
    with np.errstate(invalid="ignore"):
        return np.array([lo, hi]).astype(dtype)


def histogram(blocks, limits, shape):
    """TaskHistogram's float64 grid of numpy `shape` over `blocks` (the reference's order: binby..., expression).  Block e is binned
    along axis D-1-e.  Two dimensions: scaled = (v-min) * (1/(max-min)), kept when 0 <= scaled < 1, bin (int)(scaled*N), nothing
    at all with a non-finite limit.  More: kept when min <= v < max, bin (int)((v-min) * (N/(max-min))).  A bin that rounds up to N
    goes to N-1 and a NaN bin drops the row (where the reference writes outside its grid)."""
    D = len(blocks)
    shape = tuple(int(s) for s in shape)
    counts = np.zeros(shape, np.float64)
    if D > 3 and len(set(shape)) > 1:
        raise ValueError("histogramNd needs equal sizes")
    values = [asfloat(b) for b in blocks]
    n = len(values[0]) if values else 0
    keep = np.ones(n, bool)
    index = np.zeros(n, np.int64)
    with np.errstate(all="ignore"):
        for e, (v, (lo, hi)) in enumerate(zip(values, limits)):
            lo, hi = float(lo), float(hi)
            axis = D - 1 - e
            N = shape[axis]
            stride = int(np.prod(shape[axis + 1:], dtype=np.int64))
            if D == 2:
                if not all(np.isfinite([lo, hi])):
                    return counts
                scaled = (v - lo) * (1.0 / (hi - lo))
                ok = (scaled >= 0) & (scaled < 1)
                f = scaled * N
            else:
                ok = (v >= lo) & (v < hi)
                f = (v - lo) * (N / (hi - lo))
                ok &= ~np.isnan(f)
            b = np.minimum(np.trunc(np.where(ok, f, 0.0)), N - 1).astype(np.int64)
            keep &= ok
            index += stride * b
    np.add.at(counts.reshape(-1), index[keep], 1.0)
    return counts


def expand_shape(binby, shape, mode_shape):
    if len(binby) == 0:
        raise ValueError("only supported with binby argument given")
    try:
        len(shape)
        shape = tuple(shape)
    except TypeError:
        shape = len(binby) * (shape,)
    return (mode_shape,) + shape


def resolve(columns, expressions, value):
    """df.limits for explicit pairs and "minmax" / None, one value for all expressions or one per expression"""
    if value is None or isinstance(value, str) or np.isscalar(value[0]):
        value = [value] * len(expressions)
    return [minmax(columns[e]) if v is None or v == "minmax" else v for e, v in zip(expressions, value)]


def finish(counts, pmin, pmax, mode_shape):
    """:2022-2034 as written there"""
    indices = np.argmax(counts, axis=0)
    centers = np.linspace(pmin, pmax, mode_shape + 1)[:-1]
    centers += (centers[1] - centers[0]) / 2
    modes = centers[indices]
    ok = counts.sum(axis=0) > 0
    modes[~ok] = np.nan
    return modes


def mode(columns, expression, binby, limits=None, shape=256, mode_shape=64, mode_limits=None, selection=None, filter=None):
    binby = [binby] if isinstance(binby, str) else list(binby)
    shape = expand_shape(binby, shape, mode_shape)
    if len(shape) > 3 and len(set(shape)) > 1:
        raise ValueError("mode with three or more binby needs mode_shape equal to every binby size")
    if filter is not None:
        keep = np.asarray(columns[filter], bool)
        columns = {k: v[keep] for k, v in columns.items()}
    lims = list(resolve(columns, binby, limits)) + list(resolve(columns, [expression], mode_limits))
    blocks = [columns[e] for e in binby + [expression]]
    if selection:
        keep = np.asarray(columns[selection], bool)
        blocks = [b[keep] for b in blocks]
    counts = histogram(blocks, lims, shape)
    pmin, pmax = lims[-1]
    return finish(counts, pmin, pmax, mode_shape)


def load_golden():
    """(columns, cases): cases[name] = {"kwargs", "result" or "error", "reference": whether the compiled reference produced it}"""
    z = np.load(GOLDEN, allow_pickle=False)
    names = json.loads(str(z["names"]))
    columns = {}
    for k in json.loads(str(z["columns"])):
        data = z["col_" + k]
        columns[k] = np.ma.array(data, mask=z["mask_" + k]) if "mask_" + k in z.files else data
    cases = {}
    for name in names:
        meta = json.loads(str(z["meta_" + name]))
        if "result_" + name in z.files:
            meta["result"] = z["result_" + name]
        cases[name] = meta
    return columns, cases
