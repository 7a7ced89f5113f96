"""A minimal DataFrameLocal-shaped front over the GPU hot path, so the parity tests read like the reference's own.

Covers exactly the callers of the path (SURVEY.md section 3): ``df.count/sum/mean/std/var/min/max/first/last(binby=...,
limits=..., shape=...)`` (packages/vaex-core/vaex/dataframe.py:842-1607 -> _compute_agg), ``df.minmax/limits`` (the limits
pre-pass, dataframe.py:1519-1521, 1926-1928) and ``df.groupby(by).agg({...})`` (vaex/groupby.py, hash ordinal path).
Columns are plain arrays: numpy (host; streamed in chunks) or device arrays (torch CUDA tensors; one fused pass).
Expressions are column NAMES only — the expression system is upstream of the path and out of scope.
"""
import numpy as np

from . import _lib
from . import agg as _agg
from . import execution, taskpart
from . import hash as _hash


def _is_device(x):
    return hasattr(x, "__cuda_array_interface__") and not isinstance(x, np.ndarray)


def _dtype_of(ar):
    if _hash.is_string_column(ar):
        return np.dtype("O")
    if getattr(ar, "device_virtual", False):  # device-evaluated virtual column (hash.CombinedCodes)
        return ar.dtype
    if _is_device(ar):
        return np.dtype(ar.__cuda_array_interface__["typestr"])
    return np.asarray(ar).dtype if not np.ma.isMaskedArray(ar) else ar.dtype


class Frame:
    def __init__(self, columns, nthreads=None, executor=None, categories=None, pin=False, filter=None, variables=None):
        """pin=True page-locks the host (numpy) columns once so that chunk uploads run at PCIe rate (b200_host_register).
        filter: boolean expression string — the frame then behaves like ``df[df.<expression>]`` (dataframe.py filtered frames):
        every pass evaluates the filter on the device and compacts the dependent columns with it (vaex/execution.py:516-522)."""
        self.columns = dict(columns)
        self.variables = dict(variables or {})  # names usable inside expressions (hash maps for _ordinal_values, ...)
        self._filter_expression = filter
        self._filter = None
        self._pinned = _lib.pinned(*[v for v in self.columns.values() if isinstance(v, np.ndarray) and not np.ma.isMaskedArray(v)]) if pin else None
        self.executor = executor or execution.Executor(nthreads)
        self.categories = dict(categories or {})  # name -> (min_value, count): ordinal-coded columns (df.categorize)
        n = {len(v) for v in self.columns.values()}
        assert len(n) <= 1, "all columns must have equal length"
        self.length = n.pop() if n else 0
        if filter is not None:
            self._filter = self.expression(filter)
            if self._filter.dtype != np.bool_:
                raise ValueError(f"filter {filter!r} is not a boolean expression (dtype {self._filter.dtype})")

    def __len__(self):
        return self.length

    # ---- expressions: virtual columns, filters, selections — evaluated on the device (csrc/expr.cu) ----------------------------
    def expression(self, text):
        """compile `text` over this frame's columns into a device-evaluated column (expression.DeviceExpression)"""
        from . import expression as _expr
        real = {k: v for k, v in self.columns.items() if not isinstance(v, _expr.DeviceExpression)}
        # virtual columns are substituted textually, like vaex expands them before evaluation
        text = self._expand(str(text))
        return _expr.DeviceExpression(text, real, self.variables)

    def _expand(self, text):
        import ast
        from . import expression as _expr
        virtual = {k: v.expression for k, v in self.columns.items() if isinstance(v, _expr.DeviceExpression)}
        if not virtual:
            return text

        class Sub(ast.NodeTransformer):
            def visit_Name(self, node):
                if node.id in virtual:
                    return ast.parse("(" + virtual[node.id] + ")", mode="eval").body
                return node
        return ast.unparse(Sub().visit(ast.parse(text, mode="eval")))

    def add_virtual_column(self, name, expression):
        """df.add_virtual_column / df['name'] = expression (dataframe.py:3476-3530): evaluated on the device, never materialised"""
        self.columns[name] = self.expression(expression)

    def filter(self, expression):
        """df[df.<expression>]: a filtered view over the same columns (filters combine with &, dataframe.py:5535-5560)"""
        combined = expression if self._filter_expression is None else f"({self._filter_expression}) & ({expression})"
        f = Frame(self.columns, executor=self.executor, categories=self.categories, filter=combined, variables=self.variables)
        return f

    def evaluate(self, expression):
        """host copy of an expression's values over the whole frame (unfiltered), chunked like every other pass"""
        e = self.columns[expression] if expression in self.columns and getattr(self.columns[expression], "device_virtual", False) else self.expression(expression)
        chunk = max(self.executor.chunk_size_for(self.length), 1)
        parts = [e.chunk(0, i, min(i + chunk, self.length)).to_numpy() for i in range(0, self.length, chunk)]
        return np.concatenate(parts) if parts else np.zeros(0, e.dtype)

    def __getitem__(self, name):
        return self.columns[name]

    def dtypes(self):
        return {k: _dtype_of(v) for k, v in self.columns.items()}

    def categorize(self, name, min_value=0, count=None):
        """Mark an integer column as ordinal codes [min_value, min_value+count) -> BinnerOrdinal (dataframe.py:5605-5631)."""
        if count is None:
            lo, hi = self.minmax(name)
            min_value, count = int(lo), int(hi) - int(lo) + 1
        self.categories[name] = (int(min_value), int(count))

    # ---- legacy statistics: TaskStatistic on the device (csrc/statistic.cu) ----------------------------------------------
    def _statistic(self, op, binby, weights, limits, shape, selection, edges=False):
        """TaskStatistic(self, binby, shape, limits, weights=weights, op=op, selection=selection) (vaex/tasks.py:431-470), run
        through the executor; returns the reduced grid (one per selection when `selection` is a list)"""
        binby = [] if binby is None else ([binby] if isinstance(binby, str) else list(binby))
        shape = [shape] * len(binby) if np.isscalar(shape) else list(shape)
        if limits is None or isinstance(limits, str):
            limits = [None] * len(binby)
        limits = list(limits)
        if len(binby) == 1 and len(limits) == 2 and np.isscalar(limits[0]):
            limits = [limits]
        limits = [self.minmax(b).astype("float64") if lim is None else lim for b, lim in zip(binby, limits)]
        waslist = isinstance(selection, (list, tuple))
        selections = list(selection) if waslist else [selection]
        masks = []
        for one in selections:
            if one is None or one is False:
                masks.append(None)
                continue
            m = self.expression(one)
            if m.dtype != np.bool_:
                raise ValueError("a selection must be a boolean expression")
            masks.append(m)
        part = taskpart.TaskPartStatistic(self, [int(s) + 3 if edges else int(s) for s in shape], binby, np.dtype("f8"),
                                          [None if m is None else "selection%d" % i for i, m in enumerate(masks)], op, list(weights),
                                          [float(lim[0]) for lim in limits], [float(lim[1]) for lim in limits], edges, waslist)
        columns = dict(self.columns)
        for e in list(binby) + list(weights):
            if e not in columns:
                columns[e] = self.expression(e)
        task = execution.Task(part, masks)
        task.expressions = list(binby) + list(weights)
        self.executor.execute(columns, [task], self.length, filter=self._filter)
        return task.result

    def cov(self, x, y=None, binby=None, limits=None, shape=128, selection=None):
        """df.cov (vaex/dataframe.py:1402-1483): the covariance matrix of x and y, or of the expressions in the list x, from ONE
        fused OP_COV pass; the last two dimensions are (N, N)"""
        if y is None:
            if not isinstance(x, (list, tuple)):
                raise ValueError("if y argument is not given, x is expected to be sequence, not %r" % (x,))
            expressions = list(x)
        else:
            expressions = [x, y]
        from . import statistic as _stat
        values = self._statistic(_stat.OP_COV, binby, expressions, limits, shape, selection)
        N = len(expressions)
        counts, sums = values[..., :N], values[..., N:2 * N]
        with np.errstate(divide="ignore", invalid="ignore"):
            means = sums / counts
        meansxy = means[..., None] * means[..., None, :]
        shp = values.shape[:-1] + (N, N)
        counts = values[..., 2 * N:2 * N + N**2].reshape(shp)
        sums = values[..., 2 * N + N**2:].reshape(shp)
        with np.errstate(divide="ignore", invalid="ignore"):
            moments2 = sums / counts
        return moments2 - meansxy

    def _correlation_matrix(self, column_names, binby=None, limits=None, shape=128, selection=None):
        cov_matrix = self.cov(column_names, binby=binby, limits=limits, shape=shape, selection=selection)
        diag = np.diagonal(cov_matrix, axis1=-2, axis2=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            norm = (diag[..., np.newaxis, :] * diag[..., np.newaxis]) ** 0.5
            return cov_matrix / norm

    def correlation(self, x, y=None, binby=None, limits=None, shape=128, selection=None):
        """df.correlation (vaex/dataframe.py:1302-1373): cov[x,y] / (std[x] std[y]); a list x without y gives the correlation matrix,
        lists give arrays of pairwise results.  (The list-of-pairs form, which returns a DataFrame, is not provided.)"""
        kw = dict(binby=binby, limits=limits, shape=shape, selection=selection)
        seq = lambda v: isinstance(v, (list, tuple))  # noqa: E731
        if y is None:
            if not seq(x):
                raise ValueError("if y not given, x is expected to be a list or tuple, not %r" % (x,))
            if all(seq(k) and len(k) == 2 for k in x):
                raise NotImplementedError("correlation of a list of pairs returns a vaex DataFrame; call it per pair")
            return self._correlation_matrix(list(x), **kw)
        if seq(x) and seq(y):
            return np.array([[self.correlation(x_, y_, **kw) for y_ in y] for x_ in x])
        if seq(x):
            return np.array([self.correlation(x_, y, **kw) for x_ in x])
        if seq(y):
            return np.array([self.correlation(x, y_, **kw) for y_ in y])
        return self._correlation_matrix([x, y], **kw)[..., 0, 1]

    def covar(self, x, y, binby=None, limits=None, shape=128, selection=None):
        """df.covar (vaex/dataframe.py:1248-1299): mean(x*y) - mean(x)*mean(y) through the binned aggregations, x*y a device
        expression"""
        single = not isinstance(x, (list, tuple))
        xs, ys = ([x], [y]) if single else (list(x), list(y))
        binby_l = [] if binby is None else ([binby] if isinstance(binby, str) else list(binby))
        if binby_l and (limits is None or isinstance(limits, str)):
            limits = [self.minmax(b).astype("float64") for b in binby_l]
        out = []
        for a, b in zip(xs, ys):
            name = "(%s)*(%s)" % (a, b)
            f = Frame(dict(self.columns), executor=self.executor, categories=self.categories, filter=self._filter_expression, variables=self.variables)
            for e in (a, b):
                if e not in f.columns:
                    f.columns[e] = f.expression(e)
            f.columns[name] = f.expression(name)
            kw = dict(binby=binby_l or None, limits=limits, shape=shape, selection=selection)
            mx, my, mxy = f._agg([_agg.mean(a), _agg.mean(b), _agg.mean(name)], **kw)
            out.append(mxy - mx * my)
        return out[0] if single else np.array(out)

    # ---- limits pre-pass ---------------------------------------------------------------------------------------------
    def minmax(self, expression, raw=False, binby=None, limits=None, shape=128, selection=None):
        """df.minmax(expression): the limits pre-pass, on the device (csrc/minmax.cu).  Masked rows and NaN are ignored; like the
        reference (TaskStatistic(OP_MIN_MAX) over vaexfast.statisticNd, vaex/cpu.py:513-606) the reduction runs on the column cast
        to float64 (float64 / int64 columns) or float32 (everything else) and the (min, max) pair is cast back to the column dtype
        (vaex/dataframe.py:1524-1528).  raw=True returns the two doubles of the statistic grid.
        With `binby` (or a `selection`) the (min, max) pair is computed per bin through OP_MIN_MAX (csrc/statistic.cu); the last
        dimension of the result is 2."""
        if binby is not None or selection is not None:
            from . import statistic as _stat
            res = self._statistic(_stat.OP_MIN_MAX, binby, [expression], limits, shape, selection)
            if raw:
                return res
            col = self.columns.get(expression)
            dt = np.dtype(_dtype_of(col) if col is not None else self.expression(expression).dtype).newbyteorder("=")
            with np.errstate(invalid="ignore"):
                return res if dt.kind in "mM" else res.astype(dt)
        import ctypes as C
        col = self.columns[expression]
        ctx = _lib.context()
        out = (C.c_double * 2)()
        if getattr(col, "device_virtual", False) or self._filter is not None:
            # virtual columns and filtered frames: evaluate / compact chunk by chunk on the device, reduce every chunk
            from . import expression as _expr
            lo, hi, dt = np.inf, -np.inf, None
            chunk = max(self.executor.chunk_size_for(self.length), 1) if not all(_is_device(c) for c in getattr(col, "columns", [col])) else max(self.length, 1)
            for i1 in range(0, self.length, chunk):
                i2 = min(i1 + chunk, self.length)
                block = col.chunk(0, i1, i2) if getattr(col, "device_virtual", False) else col[i1:i2]
                if self._filter is not None:
                    if not _is_device(block) and np.ma.isMaskedArray(block):
                        raise NotImplementedError("minmax of a masked column on a filtered frame")
                    kept, (block,) = _expr.compact(0, self._filter.chunk(0, i1, i2), [block], ctx)
                    if not kept:
                        continue
                c = _lib.column(block)
                dt = c.dtype
                _lib.check(_lib.lib().b200_minmax(ctx._h, 0, c.code, c.byteswap, c.ptr, None, c.length, c.memspace, out))
                lo, hi = min(lo, out[0]), max(hi, out[1])
            res = np.array([lo, hi])
            if raw:
                return res
            dt = np.dtype(dt if dt is not None else _dtype_of(col)).newbyteorder("=")
            with np.errstate(invalid="ignore"):
                return res if dt.kind in "mM" else res.astype(dt)
        mask = None
        if not _is_device(col) and np.ma.isMaskedArray(col):
            mask = _lib.mask_column(np.ma.getmaskarray(col))
            col = np.ascontiguousarray(col.data)
        c = _lib.column(col)
        _lib.check(_lib.lib().b200_minmax(ctx._h, 0, c.code, c.byteswap, c.ptr, None if mask is None else mask.ptr, c.length, c.memspace, out))
        res = np.array([out[0], out[1]])
        if raw:
            return res
        dt = np.dtype(c.dtype).newbyteorder("=")
        if dt.kind in "mM":
            return res
        with np.errstate(invalid="ignore"):
            return res.astype(dt)

    def limits(self, expressions, value="minmax"):
        if isinstance(expressions, str):
            return self.minmax(expressions)
        return np.array([self.minmax(e) for e in expressions])

    # ---- binned statistics -------------------------------------------------------------------------------------------
    def _binner_specs(self, binby, limits, shape):
        if binby is None or binby == []:
            return []
        if isinstance(binby, (str, dict)):
            binby = [binby]
        nd = len(binby)
        shapes = [shape] * nd if np.isscalar(shape) else list(shape)
        if limits is None or isinstance(limits, str):
            limits = [None] * nd
        limits = list(limits)
        if nd == 1 and len(limits) == 2 and np.isscalar(limits[0]):
            limits = [limits]
        specs = []
        for i, b in enumerate(binby):
            if isinstance(b, dict):  # explicit spec (ordinal / hash binners)
                specs.append(b)
                continue
            dtype = _dtype_of(self.columns[b])
            if b in self.categories:
                lo, count = self.categories[b]
                specs.append({"binner-type": "ordinal", "expression": b, "dtype": dtype.str, "count": count, "minimum": lo, "invert": False})
                continue
            lim = limits[i]
            if lim is None:
                lim = self.minmax(b).astype("float64")  # the extra pass the reference runs for limits=None (dataframe.py:5618)
            specs.append({"binner-type": "scalar", "expression": b, "dtype": dtype.str, "count": int(shapes[i]), "minimum": float(lim[0]),
                          "maximum": float(lim[1])})
        return specs

    def _agg(self, aggregators, binby=None, limits=None, shape=128, selection=None, edges=False, progress=None):
        """Run several aggregators in as few passes as possible (equal binners -> one fused pass); returns their results."""
        single = not isinstance(aggregators, (list, tuple))
        aggregators = [aggregators] if single else list(aggregators)
        specs = self._binner_specs(binby, limits, shape)
        dtypes = self.dtypes()
        def as_mask(one):
            if isinstance(one, str):  # a selection expression: a boolean mask evaluated on the device per chunk
                one = self.expression(one)
                if one.dtype != np.bool_:
                    raise ValueError("a selection must be a boolean expression")
            return one
        # a LIST of selections gives one grid per selection, stacked along a new first axis (vaex/cpu.py:744-786, :798-811)
        if isinstance(selection, (list, tuple)):
            selection = [None if one is None or one is False else as_mask(one) for one in selection]
        else:
            selection = as_mask(selection)
        requests = []
        for a in aggregators:
            for prim in a.primitives():
                prim.edges = edges or prim.edges
                if isinstance(selection, list):
                    prim.selection = [None if one is None else f"selection{i}" for i, one in enumerate(selection)]
                else:
                    prim.selection = None if selection is None else "selection"
                requests.append((specs, prim, selection))
        tasks, pos = execution.merge_aggregation_tasks(requests, dtypes, self.executor.nthreads)
        self.executor.execute(self.columns, tasks, self.length, filter=self._filter, progress=progress)
        results = []
        for a in aggregators:
            grids = []
            for prim in a.primitives():
                task, k = pos[id(prim)]
                grids.append(task.result[k])
            results.append(a.combine(*grids) if isinstance(a, _agg.AggregatorDescriptorMulti) else grids[0])
        return results[0] if single else results

    def count(self, expression=None, binby=None, limits=None, shape=128, selection=None, edges=False, progress=None):
        return self._agg(_agg.count(expression or "*"), binby, limits, shape, selection, edges, progress=progress)

    def sum(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.sum(expression), binby, limits, shape, selection, edges)

    def mean(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.mean(expression), binby, limits, shape, selection, edges)

    def var(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.var(self._as_float64(expression)), binby, limits, shape, selection, edges)

    def std(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.std(self._as_float64(expression)), binby, limits, shape, selection, edges)

    def min(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.min(expression), binby, limits, shape, selection, edges)

    def max(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.max(expression), binby, limits, shape, selection, edges)

    def first(self, expression, order_expression=None, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.first(expression, order_expression), binby, limits, shape, selection, edges)

    def last(self, expression, order_expression=None, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.last(expression, order_expression), binby, limits, shape, selection, edges)

    def list(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False, dropna=False, dropnan=False, dropmissing=False):
        """df.groupby / binby with vaex.agg.list: per bin the values of `expression` (a pyarrow large_list array over the flat grid,
        first binner fastest; vaex/agg.py:654-674)"""
        return self._agg(_agg.list(expression, dropna=dropna, dropnan=dropnan, dropmissing=dropmissing), binby, limits, shape, selection, True)

    def nunique(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False, dropna=False, dropnan=False, dropmissing=False):
        """df.nunique (vaex/dataframe.py nunique -> agg.nunique -> AggNUnique_<dtype>, src/agg_nunique.cpp)."""
        return self._agg(_agg.nunique(expression, dropna=dropna, dropnan=dropnan, dropmissing=dropmissing), binby, limits, shape, selection, edges)

    def _as_float64(self, expression, columns=None):
        """var/std/skew/kurtosis run on ``expression.astype('float64')`` in the reference (vaex/agg.py:429-431, 466, 493): integer
        columns must not accumulate their powers in int64 grids.  The cast keeps the mask of a masked column (numpy's astype
        does), so masked rows stay out of count / sum / sum_moment."""
        columns = self.columns if columns is None else columns
        col = columns[expression]
        if _dtype_of(col).kind == "f":
            return expression  # float32 already accumulates in double: identical result without the cast
        name = f"astype({expression}, 'float64')"
        if _is_device(col):
            columns[name] = col.double()
        elif np.ma.isMaskedArray(col):
            columns[name] = np.ma.array(np.asarray(col.data).astype("float64"), mask=np.ma.getmaskarray(col))
        else:
            columns[name] = np.asarray(col).astype("float64")
        return name

    # ---- value_counts / unique (counter<T>, SURVEY.md 8f row 3) ----------------------------------------------------------
    def value_counts(self, expression, dropna=False, dropnan=False, dropmissing=False, ascending=False):
        """df[expression].value_counts() (vaex/cpu.py:141-283 TaskPartValueCounts over counter_<dtype>): (keys, counts) sorted by
        count; NaN / missing get their own entries unless dropped."""
        from . import superutils
        col = self.columns[expression]
        if _hash.is_string_column(col):
            # string keys: the device string set + a count per ordinal (the reference counts with counter<string>, vaex/cpu.py:141-283)
            out = self.groupby(expression, agg=[_agg.count()])
            keys, counts = np.asarray(out[expression], dtype=object), np.asarray(out["count"])
            if dropna or dropmissing:
                keep = np.array([k is not None for k in keys], dtype=bool)
                keys, counts = keys[keep], counts[keep]
            order = np.argsort(counts, kind="stable")
            order = order if ascending else order[::-1]
            return keys[order], counts[order]
        dt = _dtype_of(col)
        counter = getattr(superutils, "counter_" + np.dtype(dt).newbyteorder("=").name)(1)
        chunk = self.executor.chunk_size_for(self.length) if not _is_device(col) else max(self.length, 1)
        for i1 in range(0, self.length, chunk):
            block = col[i1:i1 + chunk]
            if not _is_device(block) and np.ma.isMaskedArray(block):
                counter.update(np.ascontiguousarray(block.data), np.ma.getmaskarray(block))
            else:
                counter.update(block if _is_device(block) else np.ascontiguousarray(block))
        keys, counts = counter.keys(), counter.counts()
        keep = [i for i, k in enumerate(keys)
                if not ((k is None and (dropna or dropmissing)) or (isinstance(k, float) and k != k and (dropna or dropnan)))]
        keys, counts = [keys[i] for i in keep], counts[keep]
        order = np.argsort(counts, kind="stable")
        if not ascending:
            order = order[::-1]
        return [keys[i] for i in order], counts[order]

    def unique(self, expression, dropna=False):
        keys, _ = self.value_counts(expression, dropna=dropna)
        return keys

    # ---- groupby ------------------------------------------------------------------------------------------------------
    def groupby(self, by, agg=None, sort=False, fused=True, combine=False):
        gb = GroupBy(self, by, sort=sort, fused=fused, combine=combine)
        return gb.agg(agg) if agg is not None else gb


class GroupBy:
    """df.groupby(key).agg(...) over hashed keys (SURVEY.md section 3.2).

    Pass 1: TaskPartHashmapUniqueCreate builds the ordered key set on the device (vaex/groupby.py:298, vaex/cpu.py:285-405).
    Pass 2: with ``fused=True`` the key column is probed inside the binby kernel (BinnerHash_*), so the ordinal column the
    reference writes and re-reads (vaex/functions.py:2454-2463 + BinnerOrdinal) never exists; ``fused=False`` reproduces
    the reference's map_ordinal -> BinnerOrdinal data flow.  Keys come out in ordinal (first-seen) order, or sorted."""

    def __init__(self, df, by, sort=False, fused=True, combine=False):
        """combine: False (dense cartesian grid over the keys' ordinals), True, or 'auto' = combine when the dense grid would hold
        fewer than 10 rows per cell (vaex/groupby.py:653-668): the keys' ordinals are fused into one int64 code on the device
        (hash.CombinedCodes) and the groupby runs over the distinct codes — the reference's sparse `_combine` path
        (vaex/groupby.py:526-584)."""
        self.by = [by] if isinstance(by, str) else list(by)
        if any(name not in df.columns for name in self.by):  # a key that is an expression: group by it as a virtual column
            df = Frame(dict(df.columns), executor=df.executor, categories=df.categories, filter=df._filter_expression, variables=df.variables)
            for name in self.by:
                if name not in df.columns:
                    df.add_virtual_column(name, name)
        self.df = df
        self.fused = fused
        self.sort = sort
        self.combined = None
        self.hash_maps = []
        for name in self.by:
            col = df.columns[name]
            part = taskpart.TaskPartHashmapUniqueCreate(None, name, _dtype_of(col), nthreads=1)
            # nthreads=1 -> 7 shards, chunks fed in row order: the ordinals of the sequential reference run
            task = execution.Task(part)
            ex = execution.Executor(1, chunk_size_max=df.executor.chunk_size_max)
            ex.execute(df.columns, [task], df.length, filter=df._filter)
            hm = task.result
            if sort:
                hm = hm.sorted()
            self.hash_maps.append(hm)
        cells = 1
        for hm in self.hash_maps:
            cells *= len(hm)
        if len(self.by) >= 2 and cells > 0 and (combine is True or (combine == "auto" and df.length / cells < 10)):
            self._combine()

    _COMBINED = "__combined_codes"

    def _combine(self):
        """vaex/groupby.py:526-584.  The keys' ordinals are fused left to right for as long as the cartesian product of the key
        counts stays below 2^63-1 (:541-548); the distinct codes of that prefix then become ONE grouper (N = the number of codes
        that occur) that is combined with the keys that are left — the reference's recursion (:572-582), here a loop.  A later
        stage reads the previous stage's codes as a device-evaluated column and looks them up in that stage's set."""
        df = self.df
        columns = [df.columns[name] for name in self.by]
        maps = list(self.hash_maps)
        self._stages = []
        while True:
            counts = [len(hm) for hm in maps]
            take, total = 1, counts[0]
            while take < len(counts) and total * counts[take] < 2 ** 63 - 1:
                total *= counts[take]
                take += 1
            if take < 2:
                raise ValueError("two key counts whose product overflows 64 bits cannot be combined")  # `assert len(combine_now) >= 2`
            # cumulative_counts (:548-556): decreasing products, the last multiplier is 1
            multipliers = [1] * take
            for i in range(take - 2, -1, -1):
                multipliers[i] = multipliers[i + 1] * counts[i + 1]
            codes = _hash.CombinedCodes(columns[:take], maps[:take], multipliers)
            part = taskpart.TaskPartHashmapUniqueCreate(None, self._COMBINED, np.dtype("int64"), nthreads=1)
            task = execution.Task(part)
            ex = execution.Executor(1, chunk_size_max=df.executor.chunk_size_max)
            ex.execute({self._COMBINED: codes}, [task], df.length, filter=df._filter)
            hm = task.result
            if self.sort:
                hm = hm.sorted()  # parents are sorted, so code order == lexicographic key order (at every stage)
            self._stages.append((codes, hm))
            if take == len(counts):
                break
            columns = [codes] + columns[take:]
            maps = [hm] + maps[take:]
        self.combined = self._stages[-1]

    def _decode(self, group_codes, level=None):
        """group code -> ordinal of every ORIGINAL key: the div/mod chain of GrouperCombined (vaex/groupby.py:352-358), unwound
        through the stages (a stage's first 'key' is the previous stage's code set)."""
        level = len(self._stages) - 1 if level is None else level
        codes, _ = self._stages[level]
        ordinals = codes.decode(group_codes)
        if level == 0:
            return ordinals
        previous = np.asarray(self._stages[level - 1][1].keys())[ordinals[0]]
        return self._decode(previous, level - 1) + ordinals[1:]

    def keys(self):
        return [hm.keys() for hm in self.hash_maps]

    def agg(self, actions):
        """actions: {column: [names]} | {column: name} | [descriptors]; returns dict of arrays (one row per non-empty group)."""
        df = self.df
        descs, labels = [], []
        columns = dict(df.columns)
        if isinstance(actions, str):  # df.groupby(by, agg='count') (vaex/groupby.py:688-700)
            actions = [_agg.aggregates[actions]("*")] if actions == "count" else {c: actions for c in df.columns if c not in self.by}
        if isinstance(actions, dict):
            for col, names in actions.items():
                if isinstance(names, _agg.AggregatorDescriptor):  # {'label': vaex.agg.mean('x')}: the key names the output column
                    descs.append(names)
                    labels.append(col)
                    continue
                for n in ([names] if isinstance(names, str) else names):
                    if isinstance(n, _agg.AggregatorDescriptor):
                        descs.append(n)
                        labels.append(f"{col}_{n.short_name}")
                        continue
                    # the moment aggregators take expression.astype('float64') like Frame.var/std do (vaex/agg.py:429-431)
                    src = df._as_float64(col, columns) if n in ("var", "std", "skew", "kurtosis") else col
                    descs.append(_agg.aggregates[n](src))
                    labels.append(f"{col}_{n}")
        else:
            for d in actions:
                descs.append(d)
                labels.append(f"{d.expressions[0] if d.expressions else 'count'}_{d.short_name}")
        descs.append(_agg.count("*"))  # the reference adds count(*) to drop empty groups (vaex/groupby.py:688-745)
        labels.append("__count")
        specs = []
        if self.combined is not None:
            codes, chm = self.combined
            columns[self._COMBINED] = codes
            frame = Frame(columns, executor=df.executor, categories=df.categories, filter=df._filter_expression, variables=df.variables)
            spec = {"binner-type": "hash", "expression": self._COMBINED, "dtype": "<i8", "hash_map_unique": chm}
            grids = frame._agg(descs, binby=[spec], edges=True)
            counts = grids[-1][:-2]
            keep = counts > 0
            group_codes = np.asarray(chm.keys())[keep]
            out = {}
            for name, hm, ordinals in zip(self.by, self.hash_maps, self._decode(group_codes)):
                out[name] = hm.keys()[ordinals]
            for label, g in zip(labels[:-1], grids[:-1]):
                out[label] = _take_cells(g, np.nonzero(keep)[0]) if _is_arrow(g) else g[:-2][keep]
            out["count"] = counts[keep]
            return out
        for name, hm in zip(self.by, self.hash_maps):
            dtype = _dtype_of(df.columns[name])
            if hm.is_string:
                cname = f"_ordinal_values({name})"
                columns[cname] = _hash.StringCodes(df.columns[name], hm)
                specs.append({"binner-type": "ordinal", "expression": cname, "dtype": "<i8", "count": len(hm), "minimum": 0, "invert": False})
            elif self.fused:
                specs.append({"binner-type": "hash", "expression": name, "dtype": dtype.str, "hash_map_unique": hm})
            else:
                codes = hm.map(df.columns[name])
                cname = f"_ordinal_values({name})"
                columns[cname] = codes
                cdt = _dtype_of(codes)
                specs.append({"binner-type": "ordinal", "expression": cname, "dtype": cdt.str, "count": len(hm), "minimum": 0, "invert": False})
        frame = Frame(columns, executor=df.executor, categories=df.categories, filter=df._filter_expression, variables=df.variables)
        grids = frame._agg(descs, binby=specs, edges=True)
        # _extract_center (vaex/groupby.py:896-977): drop the null / nan edge cells, keep groups with count > 0
        center = tuple(slice(0, -2) for _ in self.by)
        counts = grids[-1][center]
        keep = counts > 0
        out = {}
        mesh = np.meshgrid(*[np.arange(len(hm)) for hm in self.hash_maps], indexing="ij")
        for name, hm, m in zip(self.by, self.hash_maps, mesh):
            out[name] = hm.keys()[m[keep]]
        # a list aggregator returns ONE arrow list per cell of the flat FULL grid (first binner fastest, edge cells included)
        shape = [len(hm) + 2 for hm in self.hash_maps]
        strides = np.cumprod([1] + shape[:-1])
        flat = sum(i.astype(np.int64) * int(st) for i, st in zip(np.nonzero(keep), strides))
        for label, g in zip(labels[:-1], grids[:-1]):
            out[label] = _take_cells(g, flat) if _is_arrow(g) else g[center][keep]
        out["count"] = counts[keep]
        return out


def _is_arrow(x):
    return type(x).__module__.startswith("pyarrow")


def _take_cells(lists, cells):
    import pyarrow as pa
    return lists.take(pa.array(np.asarray(cells, dtype=np.int64)))
