"""percentile_approx's finish (vaex/dataframe.py:1675-1754) over a device count grid: the interpolation runs in csrc/percentile.cu
(b200_grid_percentile); the host only evaluates ``span = ub - lb`` in the limits' dtype, as numpy does in the reference, returns the
limits themselves for percentages 0 and 100, and stacks the results as the reference does."""
import ctypes as C

import numpy as np

from . import _lib


def listify(*args):
    """vaex.utils.listify: (True, args) when the first argument is a sequence, else (False, [[a] for a in args]); unpack one
    argument as ``waslist, (items,) = listify(x)``"""
    if isinstance(args[0], str):
        return False, [[x] for x in args]
    try:
        args[0][0]
        return True, args
    except Exception:
        return False, [[x] for x in args]


def unlistify(waslist, *args):
    """vaex.utils.unlistify: the inverse of listify (None for several arguments that were not lists, as there)"""
    if waslist:
        return args[0] if len(args) == 1 else args
    values = [x[0] for x in args]
    if len(values) == 1:
        return values[0]


def is_integral(p):
    """an integer percentage makes numpy multiply (total + 1) * p in int64 before the division (NEP 50)"""
    return isinstance(p, (int, np.integer, np.bool_))


def grid_percentile(grid_ptr, sizes, lb, span, percentages, ctx=None, slot=0, out=None):
    """b200_grid_percentile over the int64 device grid at `grid_ptr` (`sizes` with edges, first dimension fastest, the percentile
    axis last).  Returns a (len(percentages), cells) float64 host array, cells first binner fastest; with `out` (a device array of
    that many doubles, ``__cuda_array_interface__``) the result is written there instead."""
    ctx = ctx or _lib.context()
    sizes = [int(s) for s in sizes]
    cells = int(np.prod([s - 3 for s in sizes[:-1]], dtype=np.int64))
    n = len(percentages)
    pct = (C.c_double * max(n, 1))(*[float(p) for p in percentages])
    integral = (C.c_uint8 * max(n, 1))(*[int(is_integral(p)) for p in percentages])
    if out is None:
        host = np.empty((n, cells), np.float64)
        memspace, ptr = _lib.MEM_HOST, host.ctypes.data
    else:
        host, memspace, ptr = out, _lib.MEM_DEVICE, out.__cuda_array_interface__["data"][0]
    _lib.check(_lib.lib().b200_grid_percentile(ctx._h, ctx.slot(slot), grid_ptr, len(sizes), (C.c_int64 * len(sizes))(*sizes), float(lb), float(span),
                                               pct, integral, n, memspace, ptr))
    return host


def finish(grid_ptr, sizes, limit, percentage, ctx=None, slot=0):
    """One expression's result of the reference's finish (vaex/dataframe.py:1677-1752) from the count grid at `grid_ptr`: per
    percentage a scalar limit (0 or 100) or the grid of sliced binby cells (a numpy scalar without binby), stacked with np.array and
    unlistified over the percentages."""
    waslist, (percentages,) = listify(percentage)
    lb, ub = limit
    with np.errstate(all="ignore"):
        span = ub - lb  # in the limits' dtype: a float32 minmax gives a float32 span
    middle = [p for p in percentages if not (p == 0 or p == 100)]
    shape = tuple(int(s) - 3 for s in sizes[:-1])
    values = grid_percentile(grid_ptr, sizes, lb, span, middle, ctx, slot) if middle else None
    percentiles = []
    k = 0
    for p in percentages:
        if p == 0:
            percentiles.append(limit[0])
        elif p == 100:
            percentiles.append(limit[1])
        else:
            x = values[k].reshape(shape, order="F")
            percentiles.append(x if shape else x[()])
            k += 1
    return unlistify(waslist, np.array(percentiles))
