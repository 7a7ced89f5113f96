"""Legacy statistics on the device: the StatOp family of vaex.tasks (vaex/tasks.py:288-402) and the device grid behind
``TaskPartStatistic`` (csrc/statistic.cu, include/b200agg.h ``b200_stat_*``).

``StatOp`` restates the reference's op objects (code, fields, init, reduce) so that a part built without vaex reduces its grid
exactly like vaex does: ``nansum`` for ADD1 / COUNT / MOMENTS, ``np.sum`` for COV (a NaN product stays NaN), ``nanmin`` / ``nanmax``
for MIN_MAX and the ``argmin`` over the order field for FIRST.
"""
import ctypes as C

import numpy as np

from . import _lib


class StatOp:
    def __init__(self, code, fields=None, reduce_function=np.nansum, dtype=None):
        self.code = code
        self.fixed_fields = fields
        self.reduce_function = reduce_function
        self.dtype = dtype

    def init(self, grid):
        pass

    def fields(self, weights):
        return self.fixed_fields

    def reduce(self, grid, axis=0):
        value = self.reduce_function(grid, axis=axis)
        return value.astype(self.dtype) if self.dtype else value

    def __eq__(self, other):
        return getattr(other, "code", None) == self.code

    def __hash__(self):
        return hash(self.code)


class StatOpMinMax(StatOp):
    def init(self, grid):
        grid[..., 0] = np.inf
        grid[..., 1] = -np.inf

    def reduce(self, grid, axis=0):
        out = np.zeros(grid.shape[1:], dtype=grid.dtype)
        out[..., 0] = np.nanmin(grid[..., 0], axis=axis)
        out[..., 1] = np.nanmax(grid[..., 1], axis=axis)
        return out


class StatOpCov(StatOp):
    def __init__(self, code, fields=None, reduce_function=np.sum):
        super().__init__(code, fields, reduce_function=reduce_function)

    def fields(self, weights):
        n = len(weights)
        return n * 2 + n**2 * 2


class StatOpFirst(StatOp):
    def __init__(self, code, fields=2, reduce_function=None):
        super().__init__(code, 2, reduce_function=self._reduce_function)

    def init(self, grid):
        grid[..., 0] = np.nan
        grid[..., 1] = np.inf

    def _reduce_function(self, grid, axis=0):
        values = grid[..., 0]
        indices = np.argmin(grid[..., 1], axis=0)
        if len(values.shape) == 2:
            return values[indices, np.arange(values.shape[1])[:, None]][0]
        if len(values.shape) == 3:
            return values[indices, np.arange(values.shape[1])[:, None], np.arange(values.shape[2])]
        if len(values.shape) == 4:
            return values[indices, np.arange(values.shape[1])[:, None], np.arange(values.shape[2])[None, :, None], np.arange(values.shape[3])]
        raise ValueError("dimension %d not yet supported" % len(values.shape))


OP_ADD1 = StatOp(0, 1)
OP_COUNT = StatOp(1, 1)
OP_MIN_MAX = StatOpMinMax(2, 2)
OP_ADD_WEIGHT_MOMENTS_01 = StatOp(3, 2, np.nansum)
OP_ADD_WEIGHT_MOMENTS_012 = StatOp(4, 3, np.nansum)
OP_COV = StatOpCov(5)
OP_FIRST = StatOpFirst(6)


def decode_op(spec):
    """the '_op' encoding of vaex/tasks.py:375-393"""
    spec = dict(spec)
    if "reduce_function" in spec:
        spec["reduce_function"] = getattr(np, spec.pop("reduce_function"))
    cls = {2: StatOpMinMax, 5: StatOpCov, 6: StatOpFirst}.get(spec["code"], StatOp)
    return cls(**spec)


def compute_class(dtypes):
    """vaex/cpu.py:527-541: float64 and int64 (alone or as the common type) compute in float64, everything else in float32"""
    dtype = np.result_type(*dtypes)
    return _lib.F64 if dtype.kind == "f" and dtype.itemsize == 8 or dtype.kind == "i" and dtype.itemsize == 8 else _lib.F32


class StatColumn(C.Structure):
    _fields_ = [("data", C.c_void_p), ("dtype", C.c_int32), ("byteswap", C.c_int32), ("mask", C.c_void_p)]


class Statistic:
    """One device grid of a statistic: ``bin`` chunks into it (any slot, any thread), ``read`` the reference's double grid
    (nselections, *sizes, fields)."""

    def __init__(self, op_code, cls, sizes, minima, maxima, edges, nweights, nselections, ctx=None):
        self.ctx = ctx or _lib.context()
        self.sizes = tuple(int(s) for s in sizes)
        self.nselections = int(nselections)
        nd = len(self.sizes)
        h = C.c_void_p()
        _lib.check(_lib.lib().b200_stat_create(self.ctx._h, int(op_code), int(cls), nd, (C.c_int64 * max(nd, 1))(*self.sizes),
                                               (C.c_double * max(nd, 1))(*[float(v) for v in minima]),
                                               (C.c_double * max(nd, 1))(*[float(v) for v in maxima]), int(bool(edges)), int(nweights),
                                               self.nselections, C.byref(h)))
        self._h = h
        self.fields = _lib.lib().b200_stat_fields(h)
        # slot -> the device blocks of that slot's last call: the kernel reads them after `bin` returns, so they are held until the
        # slot's next call has waited for its stream (or until `read` / `reset` / `close`, which wait for every slot)
        self._held = {}

    def bin(self, slot, binby, weights, selections, nrows, row_offset):
        """binby / weights: arrays (numpy, numpy.ma or device); selections: one entry per selection, None = all rows.
        row_offset: the global index of the block's first row; FIRST breaks ties by it, so every row of a pass needs its own."""
        keep = []

        def column(ar):
            ar, mask = _lib.split_mask(ar)
            if mask is not None:
                mask = _lib.mask_column(mask)
            if _lib.dtype_of(ar).kind in "mM":  # the signed count of units, as numpy's astype(float) reads it
                ar = _lib.int64_view(ar)
            c = _lib.column(ar)
            if c.length != nrows:
                raise RuntimeError(f"expected a block of {nrows} rows, got {c.length}")
            keep.extend([c, mask])
            return StatColumn(c.ptr, c.code, c.byteswap, None if mask is None else mask.ptr)

        b = (StatColumn * max(len(binby), 1))(*[column(a) for a in binby])
        w = (StatColumn * max(len(weights), 1))(*[column(a) for a in weights])
        sel = (C.c_void_p * self.nselections)()
        for i, s in enumerate(selections):
            if s is not None:
                m = _lib.mask_column(s)
                keep.append(m)
                sel[i] = m.ptr
        memspace = _lib.memspace(*keep)
        slot = self.ctx.slot(0 if slot is None else slot)
        if self._held.pop(slot, None) is not None:
            self.ctx.sync(slot)  # the previous call's kernel on this slot is done with its blocks
        _lib.check(_lib.lib().b200_stat_bin(self._h, slot, b, w, sel, int(nrows), int(row_offset), memspace, 0))
        if memspace == _lib.MEM_DEVICE:  # HOST blocks were copied during the call, MIXED calls wait for their stream
            self._held[slot] = keep

    def read(self):
        out = np.empty((self.nselections,) + self.sizes + (self.fields,), np.float64)
        _lib.check(_lib.lib().b200_stat_read(self._h, out.ctypes.data))  # waits for every slot
        self._held.clear()
        return out

    def reset(self):
        _lib.check(_lib.lib().b200_stat_reset(self._h))  # waits for every slot
        self._held.clear()

    def close(self):
        if self._h:
            _lib.lib().b200_stat_destroy(self._h)  # waits for every slot
            self._h = None
        self._held.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

