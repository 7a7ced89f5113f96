"""mutual_information (vaex/dataframe.py:685-819): the planning of the combinations (:730-763), the finish of every count grid on the
device (csrc/mutinfo.cu, b200_grid_mutual_information) and the assembly of the result (:804-817).  Frame.mutual_information runs the
count passes; this module holds what the reference computes around them, so that a caller with its own count grid in device memory
(for example after ``engine.all_reduce``) can finish it the same way."""
import ctypes as C
import itertools

import numpy as np

from . import _lib
from .frame import _issequence
from .percentile import listify, unlistify

# the count grids of one executor pass stay under this share of the device's free memory; GRID_BUDGET_BYTES, when set, caps it
GRID_BUDGET_FRACTION = 0.5
GRID_BUDGET_BYTES = None


def plan(x, y=None, dimension=2, mi_limits=None):
    """The argument forms of :730-760 -> (combinations, shape_result, waslist, mi_limits): a list of tuples of length 2, a matrix of
    `dimension` axes over x, the x by y matrix, x against one y, or one pair.  For one pair `mi_limits` comes back wrapped as
    [mi_limits].  A single string x with a list y pairs every character of x with the list, which fails later as it does there."""
    if y is None and _issequence(x) and all(_issequence(k) for k in x):
        waslist, (combinations,) = listify(x)
        shape_result = (len(combinations),)
    elif _issequence(x) and (_issequence(y) or y is None):
        if y is None:
            combinations = list(itertools.product(x, repeat=dimension))
            shape_result = (len(x),) * dimension
        else:
            shape_result = (len(x), len(y))
            combinations = np.array([[(i, j) for i in y] for j in x]).reshape((-1, 2)).tolist()
        waslist = True
    elif _issequence(x):
        shape_result = (len(x),)
        combinations = [(i, y) for i in x]
        waslist = True
    elif _issequence(y):
        shape_result = (len(y),)
        combinations = [(i, y) for i in x]
        waslist = True
    else:
        shape_result = tuple()
        combinations = [(x, y)]
        waslist = False
        if mi_limits:
            mi_limits = [mi_limits]
    return combinations, shape_result, waslist, mi_limits


def unique_combinations(combinations):
    """every combination sorted, then np.unique over them (:765-768): (unique combinations as tuples, inverse index)"""
    combinations_sorted = [tuple(sorted(k)) for k in combinations]
    combinations_unique, unique_reverse = np.unique(combinations_sorted, return_inverse=True, axis=0)
    return list(map(tuple, combinations_unique.tolist())), unique_reverse


def assemble(mi_list, x, unique_reverse, binby_shape, shape_result, waslist, sort):
    """`finish` (:804-817): with sort, the unique combinations' values sorted descending and x indexed by those positions; else
    the values in the caller's order, reshaped (not transposed) to binby_shape + shape_result"""
    mi_list = np.array(mi_list)
    if sort:
        indices = np.argsort(mi_list)[::-1]
        sorted_x = [x[k] for k in indices]  # first, as there: with binby this raises TypeError
        return mi_list[indices], sorted_x
    mi_list = mi_list[unique_reverse]
    return np.array(unlistify(waslist, mi_list)).reshape(tuple(binby_shape) + tuple(shape_result))


def grid_mutual_information(grid_ptr, sizes, dimension, ctx=None, slot=0, out=None):
    """b200_grid_mutual_information over the int64 device grid at `grid_ptr` (`sizes` with edges, first dimension fastest, the
    `dimension` MI axes first).  Returns one float64 per sliced binby cell, first binner fastest, in a host array; with `out` (a
    device array of that many doubles, ``__cuda_array_interface__``) the result is written there instead."""
    ctx = ctx or _lib.context()
    sizes = [int(s) for s in sizes]
    cells = int(np.prod([s - 3 for s in sizes[dimension:]], dtype=np.int64))
    if out is None:
        host = np.empty(cells, np.float64)
        memspace, ptr = _lib.MEM_HOST, host.ctypes.data
    else:
        host, memspace, ptr = out, _lib.MEM_DEVICE, out.__cuda_array_interface__["data"][0]
    _lib.check(_lib.lib().b200_grid_mutual_information(ctx._h, ctx.slot(slot), grid_ptr, len(sizes), (C.c_int64 * len(sizes))(*sizes),
                                                       int(dimension), memspace, ptr))
    return host


def finish(grid_ptr, sizes, dimension, ctx=None, slot=0):
    """`calculate` (:766-790) of one combination's count grid: a float64 scalar without binby, else the binby grid"""
    values = grid_mutual_information(grid_ptr, sizes, dimension, ctx, slot)
    shape = tuple(int(s) - 3 for s in sizes[dimension:])
    return values.reshape(shape, order="F") if shape else values[0]


def grid_budget(device):
    """bytes of count grid one executor pass may hold, and the device's free bytes"""
    import torch
    free, _ = torch.cuda.mem_get_info(device)
    budget = int(free * GRID_BUDGET_FRACTION)
    if GRID_BUDGET_BYTES is not None:
        budget = min(budget, int(GRID_BUDGET_BYTES))
    return budget, free


def batches(nbytes, budget):
    """consecutive groups of grid sizes whose sum stays under `budget`; a grid larger than the budget runs alone"""
    out, current, held = [], [], 0
    for i, n in enumerate(nbytes):
        if current and held + n > budget:
            out.append(current)
            current, held = [], 0
        current.append(i)
        held += n
    if current:
        out.append(current)
    return out
