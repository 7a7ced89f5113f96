"""df.mode (vaex/dataframe.py:2006-2034): the planning of the legacy histogram it counts (vaex.legacy.TaskHistogram,
vaex/legacy.py:22-110, over vaexfast histogram2d / histogram3d / histogramNd) and the argmax finish on the device
(csrc/statistic.cu, b200_stat_create_histogram / b200_stat_mode).  Frame.mode runs the count pass; this module holds what the
reference computes around it."""
import ctypes as C

import numpy as np

from . import _lib
from . import statistic as _stat


def grid_shape(binby, shape=256, mode_shape=64):
    """the histogram's numpy shape (mode_shape,) + one size per binby (:2009-2017).  vaexfast bins its first block along the last
    axis, so the expression lands on axis 0 and the first binby on the last axis.  histogramNd (three or more binby) scales each
    block by the size of one axis and strides it by another: only equal sizes give the grid the reference means."""
    if len(binby) == 0:
        raise ValueError("only supported with binby argument given")
    try:
        len(shape)
        shape = tuple(shape)
    except TypeError:
        shape = len(binby) * (shape,)
    shape = tuple(int(s) for s in (mode_shape,) + tuple(shape))
    if len(shape) > 3 and len(set(shape)) > 1:
        raise ValueError(f"mode with {len(binby)} binby expressions needs mode_shape equal to every binby size (got {shape}): the "
                         "reference's histogramNd scales each axis by another axis's size, which is only correct when they agree")
    return shape


def axis_order(blocks):
    """the reference's blocks (binby..., expression) in grid axis order, axis 0 first"""
    return list(blocks)[::-1]


def centers(pmin, pmax, mode_shape):
    """the bin centers of the mode axis, numpy's own expression (:2025-2026); mode_shape 1 raises IndexError as there"""
    c = np.linspace(pmin, pmax, mode_shape + 1)[:-1]
    c += (c[1] - c[0]) / 2
    return c


def grid_bytes(shape):
    return 8 * int(np.prod(shape, dtype=np.int64))


def check_memory(shape, device):
    """MemoryError before anything is allocated when the count grid cannot fit the device's free memory"""
    from .mutual_information import grid_budget
    _, free = grid_budget(device)
    nbytes = grid_bytes(shape)
    if nbytes > free:
        raise MemoryError(f"mode: the count grid of shape {tuple(shape)} ({nbytes} bytes) exceeds the {free} bytes free on the device")


class Histogram(_stat.Statistic):
    """One device histogram of vaexfast's legacy bin rules: ``bin`` chunks into it like a Statistic (columns in grid axis order),
    ``read`` the counts as the reference's float64 grid, ``mode`` the argmax finish."""

    def __init__(self, sizes, minima, maxima, ctx=None):
        self.ctx = ctx or _lib.context()
        self.sizes = tuple(int(s) for s in sizes)
        self.nselections = 1
        nd = len(self.sizes)
        h = C.c_void_p()
        self._h = None
        self._held = {}
        _lib.check(_lib.lib().b200_stat_create_histogram(self.ctx._h, nd, (C.c_int64 * nd)(*self.sizes),
                                                         (C.c_double * nd)(*[float(v) for v in minima]),
                                                         (C.c_double * nd)(*[float(v) for v in maxima]), C.byref(h)))
        self._h = h
        self.fields = 1

    def read(self):
        return super().read()[0, ..., 0]

    def mode(self, centers):
        """per cell of axes 1.. the center of the first largest count along axis 0, NaN for an empty cell; in centers' dtype"""
        centers = np.asarray(centers)
        c = np.ascontiguousarray(centers, dtype=np.float64)
        if len(c) != self.sizes[0]:
            raise ValueError(f"{len(c)} centers for a mode axis of {self.sizes[0]} bins")
        out = np.empty(self.sizes[1:], np.float64)
        _lib.check(_lib.lib().b200_stat_mode(self._h, c.ctypes.data, out.ctypes.data))  # waits for every slot
        self._held.clear()
        return out.astype(centers.dtype, copy=False)
