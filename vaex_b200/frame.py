"""A minimal DataFrameLocal-shaped front over the GPU hot path, so the parity tests read like the reference's own.

Covers exactly the callers of the path (SURVEY.md section 3): ``df.count/sum/mean/std/var/min/max/first/last(binby=...,
limits=..., shape=...)`` (packages/vaex-core/vaex/dataframe.py:842-1607 -> _compute_agg), ``df.minmax/limits`` (the limits
pre-pass, dataframe.py:1519-1521, 1926-1928) and ``df.groupby(by).agg({...})`` (vaex/groupby.py, hash ordinal path).
Columns are plain arrays: numpy (host; streamed in chunks) or device arrays (torch CUDA tensors; one fused pass).
Expressions are column NAMES only — the expression system is upstream of the path and out of scope.
"""
import ast
import collections
import re

import numpy as np

from . import _lib
from . import agg as _agg
from . import execution, selections, taskpart
from . import hash as _hash
from .groupby import Binner, BinnerBase, BinnerInteger, BinnerTime  # noqa: F401  (vaex.groupby's binners, for Frame.groupby)


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
        # named selections (vaex/dataframe.py:205-206): per name a history of selection objects and the index of the current one
        self.selection_histories = collections.defaultdict(list)
        self.selection_history_indices = collections.defaultdict(lambda: -1)
        if filter is not None:
            self._filter = self.expression(filter)
            if self._filter.dtype != np.bool_:
                raise ValueError(f"filter {filter!r} is not a boolean expression (dtype {self._filter.dtype})")

    def __len__(self):
        return self.length

    def _derive(self, columns, filter=None, drop_filter=False):
        """a frame over `columns` with this frame's executor, categories, variables and, unless `filter` is given or `drop_filter` is
        true, its filter; the filter is compiled again because a compiled expression is bound to its frame's column dict"""
        if filter is None and not drop_filter:
            filter = self._filter_expression
        f = Frame(columns, executor=self.executor, categories=self.categories, filter=filter, variables=self.variables)
        # a copy of the selection histories, as vaex's copy() takes (vaex/dataframe.py:3293-3298)
        for name, history in self.selection_histories.items():
            f.selection_histories[name] = list(history)
        f.selection_history_indices.update(self.selection_history_indices)
        return f

    def _with_columns(self, names):
        """this frame when every name is one of its columns, else a derived frame in which each missing name is a device-evaluated
        column"""
        missing = [e for e in dict.fromkeys(names) if e not in self.columns]
        if not missing:
            return self
        f = self._derive(self.columns)
        for e in missing:
            f.columns[e] = f.expression(e)
        return f

    def _selection(self, selection, memo=None):
        """a selection argument -> None for None / False, a boolean device expression for a string, a mask array as it is, and a
        list of selections element by element.  True means the selection named "default"; a string that names selections of this
        frame (and no column) is resolved through them (selections.resolve_text), every name to one object within the call."""
        if isinstance(selection, (list, tuple)):
            memo = {} if memo is None else memo
            return [self._selection(one, memo) for one in selection]
        if selection is None or selection is False:
            return None
        if selection is True:
            return _boolean_selection(selections.resolve_text(self, "default", memo))
        if isinstance(selection, str):
            try:
                mask = self.expression(selection)
            except KeyError:
                if not selections.names_selection(self, selection):
                    raise
                mask = selections.resolve_text(self, selection, memo)
            return _boolean_selection(mask)
        return selection

    # ---- named selections (vaex/dataframe.py:5000-5303), evaluated on the device (vaex_b200/selections.py) ------------------------
    def get_selection(self, name="default"):
        """the current selection object of `name`, None when there is none"""
        name = "default" if name is True else name
        history = self.selection_histories[name]
        index = self.selection_history_indices[name]
        return None if index == -1 else history[index]

    def has_selection(self, name="default"):
        return self.get_selection(name) is not None

    def _has_history(self, name):
        """whether `name` is a selection of this frame that selects something, without adding an empty history for it"""
        return bool(self.selection_histories.get(name)) and self.get_selection(name) is not None

    def selection_can_undo(self, name="default"):
        return self.selection_history_indices[name] > -1

    def selection_can_redo(self, name="default"):
        return (self.selection_history_indices[name] + 1) < len(self.selection_histories[name])

    def selection_undo(self, name="default"):
        if not self.selection_can_undo(name=name):
            raise ValueError(f"selection {name!r} has nothing to undo")
        self.selection_history_indices[name] -= 1

    def selection_redo(self, name="default"):
        if not self.selection_can_redo(name=name):
            raise ValueError(f"selection {name!r} has nothing to redo")
        self.selection_history_indices[name] += 1

    def _push_selection(self, create, name, check=True):
        """DataFrame._selection (vaex/dataframe.py:5285-5299): the new entry goes after the current one and the redo tail is clipped.
        The current entry is the reference's: with the index at -1 and a non-empty history that is the LAST entry.  `check`
        resolves the new entry first, so a selection that cannot be evaluated is refused before it is recorded."""
        history = self.selection_histories[name]
        current = history[self.selection_history_indices[name]] if history else None
        selection = create(current)
        if check and selection is not None:
            _boolean_selection(selections.resolve(self, selection, stack=(name,)))
        history.append(selection)
        self.selection_history_indices[name] += 1
        del history[self.selection_history_indices[name]:-1]

    def select(self, boolean_expression, mode="replace", name="default"):
        """df.select (vaex/dataframe.py:5041-5059): select by a boolean expression, combined with the current selection of `name` by
        `mode` (replace / and / or / xor / subtract).  None clears the selection (and records nothing when there is none)."""
        if boolean_expression is not None:
            boolean_expression = str(boolean_expression)
        if boolean_expression is None and not self.has_selection(name=name):
            return
        self._push_selection(lambda current: selections.SelectionExpression(boolean_expression, current, mode) if boolean_expression else None, name)

    def select_nothing(self, name="default"):
        self.select(None, name=name)

    def select_rectangle(self, x, y, limits, mode="replace", name="default"):
        self.select_box([x, y], limits, mode=mode, name=name)

    def select_box(self, spaces, limits, mode="replace", name="default"):
        """df.select_box (vaex/dataframe.py:5156-5173): the reference's text, each limit written with %f"""
        self.select(selections.box_text(spaces, limits), mode=mode, name=name)

    def select_circle(self, x, y, xc, yc, r, mode="replace", name="default", inclusive=True):
        """df.select_circle (vaex/dataframe.py:5175-5199); the squares are written as products (selections.Text)"""
        self.select(selections.circle_text(x, y, xc, yc, r, inclusive).device, mode=mode, name=name)

    def select_ellipse(self, x, y, xc, yc, width, height, angle=0, mode="replace", name="default", radians=False, inclusive=True):
        """df.select_ellipse (vaex/dataframe.py:5201-5242); the squares are written as products (selections.Text)"""
        text = selections.ellipse_text(x, y, xc, yc, width, height, angle, radians=radians, inclusive=inclusive)
        self.select(text.device, mode=mode, name=name)

    def select_lasso(self, expression_x, expression_y, xsequence, ysequence, mode="replace", name="default"):
        """df.select_lasso (vaex/dataframe.py:5244-5259): the rows whose (x, y) lie inside the polygon, tested on the device
        (b200_lasso); a row with a masked x or y is never selected"""
        self._push_selection(lambda current: selections.SelectionLasso(expression_x, expression_y, xsequence, ysequence, current, mode), name)

    def select_inverse(self, name="default"):
        """df.select_inverse (vaex/dataframe.py:5261-5271); without a selection to invert it raises and records nothing"""
        history = self.selection_histories[name]
        if (history[self.selection_history_indices[name]] if history else None) is None:
            raise ValueError(f"select_inverse: there is no selection {name!r} to invert")
        self._push_selection(selections.SelectionInvert, name)

    def select_non_missing(self, drop_nan=True, drop_masked=True, column_names=None, mode="replace", name="default"):
        """df.select_non_missing (vaex/dataframe.py:5061-5077): the rows with no NaN (drop_nan) and no missing value (drop_masked:
        masked, arrow null, None) in any of `column_names`, by default every real column"""
        from . import expression as _expr
        column_names = column_names or [k for k, v in self.columns.items() if not isinstance(v, _expr.DeviceExpression)]
        self._push_selection(lambda current: selections.SelectionDropNa(drop_nan, drop_masked, [str(k) for k in column_names], current, mode), name)

    def set_selection(self, selection, name="default"):
        self._push_selection(lambda current: selection, name)

    def selected_length(self, selection="default"):
        """the number of rows the selection selects (vaex/dataframe.py:7122-7124)"""
        return int(np.asarray(self.count(selection=selection)).item())

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
        return self._derive(self.columns, expression if self._filter_expression is None else f"({self._filter_expression}) & ({expression})")

    def evaluate(self, expression):
        """host copy of an expression's values over the whole frame (unfiltered), chunked like every other pass"""
        e = self.columns[expression] if expression in self.columns and getattr(self.columns[expression], "device_virtual", False) else self.expression(expression)
        chunk = max(self.executor.chunk_size_for(self.length), 1)
        parts = [e.chunk(0, i, min(i + chunk, self.length)).to_numpy() for i in range(0, self.length, chunk)]
        return np.concatenate(parts) if parts else np.zeros(0, e.dtype)

    def __getitem__(self, name):
        return self.columns[name]

    def dtypes(self):
        return {k: _lib.dtype_of(v) for k, v in self.columns.items()}

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
        binby, shape, limits = _binned_args(binby, shape, limits)
        limits = [self.minmax(b).astype("float64") if lim is None else lim for b, lim in zip(binby, limits)]
        waslist = isinstance(selection, (list, tuple))
        masks = self._selection(selection) if waslist else [self._selection(selection)]
        part = taskpart.TaskPartStatistic(self, [int(s) + 3 if edges else int(s) for s in shape], binby, np.dtype("f8"),
                                          [None if m is None else "selection%d" % i for i, m in enumerate(masks)], op, list(weights),
                                          [float(lim[0]) for lim in limits], [float(lim[1]) for lim in limits], edges, waslist)
        f = self._with_columns(binby + list(weights))
        task = execution.Task(part, masks)
        task.expressions = binby + list(weights)
        f.executor.execute(f.columns, [task], f.length, filter=f._filter)
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
        binby_l = _binned_args(binby, shape, limits)[0]
        if binby_l and (limits is None or isinstance(limits, str)):
            limits = [self.minmax(b).astype("float64") for b in binby_l]
        out = []
        for a, b in zip(xs, ys):
            name = "(%s)*(%s)" % (a, b)
            f = self._with_columns([a, b, name])
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
            return _minmax_as(res, _lib.dtype_of(col) if col is not None else self.expression(expression).dtype)
        import ctypes as C
        col = self.columns[expression]
        ctx = _lib.context()
        out = (C.c_double * 2)()
        if getattr(col, "device_virtual", False) or self._filter is not None:
            # virtual columns and filtered frames: evaluate / compact chunk by chunk on the device, reduce every chunk
            from . import expression as _expr
            lo, hi, dt = np.inf, -np.inf, None
            chunk = max(self.executor.chunk_size_for(self.length), 1) if not _lib.on_device(col) else max(self.length, 1)
            for i1 in range(0, self.length, chunk):
                i2 = min(i1 + chunk, self.length)
                block = _lib.chunk_of(col, 0, i1, i2)
                if self._filter is not None:
                    if not _lib.is_device(block) and np.ma.isMaskedArray(block):
                        raise NotImplementedError("minmax of a masked column on a filtered frame")
                    kept, (block,) = _expr.compact(0, self._filter.chunk(0, i1, i2), [block], ctx)
                    if not kept:
                        continue
                c = _lib.column(block)
                dt = c.dtype
                _lib.check(_lib.lib().b200_minmax(ctx._h, 0, c.code, c.byteswap, c.ptr, None, c.length, c.memspace, out))
                lo, hi = min(lo, out[0]), max(hi, out[1])
            res = np.array([lo, hi])
            return res if raw else _minmax_as(res, dt if dt is not None else _lib.dtype_of(col))
        col, mask = _lib.split_mask(col)
        mask = None if mask is None else _lib.mask_column(mask)
        c = _lib.column(col)
        _lib.check(_lib.lib().b200_minmax(ctx._h, 0, c.code, c.byteswap, c.ptr, None if mask is None else mask.ptr, c.length, c.memspace, out))
        res = np.array([out[0], out[1]])
        return res if raw else _minmax_as(res, c.dtype)

    def limits(self, expressions, value="minmax", selection=None):
        """df.limits (vaex/dataframe.py:1844-2004): the (min, max) pair `value` describes per expression: "minmax", "N%"
        (limits_percentage) or an explicit pair, returned as given.  `value` may also hold one of those per expression."""
        if isinstance(expressions, str):
            return self._limit(expressions, value, selection)
        return np.array(self._limits_list(expressions, value, selection))

    def _limits_list(self, expressions, value, selection, memo=None):
        """one limit per expression; with `memo` (a dict kept over one call), an expression's "minmax" / "N%" limit is computed
        once however many lists name it, as vaex keys its limit tasks by (expression, value) (vaex/dataframe.py:1903-1905)"""
        values = _per_expression("minmax" if value is None else value, len(expressions))
        out = []
        for e, v in zip(expressions, values):
            if memo is None or _is_limit(v) or not isinstance(v, (str, type(None))):
                out.append(self._limit(e, v, selection))
                continue
            key = (e, "minmax" if v is None else v, selection)
            if key not in memo:
                memo[key] = self._limit(e, v, selection)
            out.append(memo[key])
        return out

    def _limit(self, expression, value, selection=None):
        if _is_limit(value):
            return value
        if value is None or value == "minmax":
            return self.minmax(expression, selection=selection)
        match = re.match(r"([\d.]*)(\D*)", value)
        number, kind = match.groups()
        if kind.strip() in ("%", "percent"):
            return self.limits_percentage(expression, ast.literal_eval(number), selection=selection)
        raise NotImplementedError(f"limits {value!r}: only 'minmax', 'N%' and explicit [min, max] pairs are supported")

    def bin_edges(self, expression, limits, shape=128):
        """df.bin_edges (vaex/dataframe.py:821-822): the shape + 1 edges of `shape` equal bins over `limits`"""
        return self.bins(expression, limits, shape=shape, edges=True)

    def bin_centers(self, expression, limits, shape=128):
        """df.bin_centers (vaex/dataframe.py:824-825): the centers of `shape` equal bins over `limits`"""
        return self.bins(expression, limits, shape=shape, edges=False)

    def bins(self, expression, limits, shape=128, edges=True):
        """df.bins (vaex/dataframe.py:827-835), numpy only: the bin edges, or the bin centers with edges=False"""
        if edges:
            return np.ogrid[limits[0]:limits[1]:(shape + 1) * 1j]
        dx = (limits[1] - limits[0]) / shape
        return np.ogrid[limits[0]:limits[1] - dx:(shape) * 1j] + dx / 2

    def limits_percentage(self, expression, percentage=99.73, square=False, selection=None):
        """df.limits_percentage (vaex/dataframe.py:1795-1842): a range around the median holding about `percentage` % of the rows, read
        off the normalised cumulative counts of a 16384-bin count between the minmax limits (np.interp on the host)"""
        from . import percentile as _pct
        waslist, (expressions,) = _pct.listify(expression)
        out = []
        for e in expressions:
            limits_minmax = self.minmax(e, selection=selection)
            vmin, vmax = limits_minmax
            size = 1024 * 16
            counts = self.count(binby=e, shape=size, limits=limits_minmax, selection=selection)
            cumcounts = np.concatenate([[0], np.cumsum(counts)])
            cumcounts = cumcounts / cumcounts.max()
            f = (1 - percentage / 100.) / 2
            x = np.linspace(vmin, vmax, size + 1)
            out.append(np.interp([f, 1 - f], cumcounts, x))
        return _pct.unlistify(waslist, out)

    # ---- approximate percentiles: one count pass, the finish on the device (csrc/percentile.cu) -----------------------------
    def percentile_approx(self, expression, percentage=50., binby=None, limits=None, shape=128, percentile_shape=1024, percentile_limits="minmax",
                          selection=None):
        """df.percentile_approx (vaex/dataframe.py:1632-1780): the percentile(s) `percentage` of one expression or a list, optionally per
        cell of a binby grid, interpolated in the cumulative counts of a `percentile_shape`-bin count between `percentile_limits` (one
        pair or "minmax" / "N%" for all expressions, or one per expression).  Every expression's count grid is built in the same pass
        and finished on the device.  With two or more binby dimensions each cell gets the answer of the reference's one-dimensional
        code for that cell (DESIGN.md section 3)."""
        from . import percentile as _pct
        waslist, (expressions,) = _pct.listify(expression)
        expressions = [str(e) for e in expressions]
        binby = [] if binby is None else ([binby] if not isinstance(binby, (list, tuple)) else list(binby))
        selection = None if selection is False else selection
        shape = _expand_shape(shape, len(binby))
        percentile_shapes = _expand_shape(percentile_shape, len(expressions))
        if percentile_limits:
            percentile_limits = _expand_limits(percentile_limits, len(expressions))
        f = self._with_columns(expressions + binby)
        for e in expressions + binby:
            if e in f.categories or _lib.dtype_of(f.columns[e]).kind in "mM":
                raise NotImplementedError(f"percentile_approx over the categorical or datetime column {e!r} is not supported")
        binby_limits = f._limits_list(binby, limits, selection)
        expression_limits = f._limits_list(expressions, percentile_limits, selection)
        mask = f._selection(selection)
        dtypes = f.dtypes()
        tasks = []
        for e, pshape, plim in zip(expressions, percentile_shapes, expression_limits):
            specs = [_scalar_spec(b, dtypes[b], n, lim) for b, n, lim in zip(binby, shape, binby_limits)]
            specs.append(_scalar_spec(e, dtypes[e], pshape, plim))
            part = taskpart.TaskPartCountGrid("percentile_approx", specs, mask is not None, dtypes, _pct.finish, (plim, percentage), f.executor.nthreads)
            tasks.append(execution.Task(part, [mask]))
        f.executor.execute(f.columns, tasks, f.length, filter=f._filter)
        return _pct.unlistify(waslist, np.array([t.result for t in tasks]))

    def median_approx(self, expression, percentage=50., binby=None, limits=None, shape=128, percentile_shape=256, percentile_limits="minmax",
                      selection=None):
        """df.median_approx (vaex/dataframe.py:1611-1629): percentile_approx at the integer percentage 50 (`percentage` is ignored, as
        there), 256 percentile bins by default"""
        return self.percentile_approx(expression, 50, binby=binby, limits=limits, shape=shape, percentile_shape=percentile_shape,
                                      percentile_limits=percentile_limits, selection=selection)

    # ---- mutual information: count passes, the per-cell finish on the device (csrc/mutinfo.cu) --------------------------------
    def mutual_information(self, x, y=None, dimension=2, mi_limits=None, mi_shape=256, binby=[], limits=None, shape=128, sort=False,
                           selection=False):
        """df.mutual_information (vaex/dataframe.py:685-819) between x and y, a list of pairs, a `dimension`-axis matrix over x or the
        x by y matrix, on an `mi_shape` grid between `mi_limits`, optionally per cell of a binby grid (at most 3 axes).  Every unique
        combination is one count(*) grid finished on the device; the combinations of a call share executor passes, as many per pass
        as fit the grid budget of mutual_information.py.  The reference's result shapes and quirks are kept (DESIGN.md section 3);
        a string `binby` is one expression."""
        from . import mutual_information as _mi
        combinations, shape_result, waslist, mi_limits = _mi.plan(x, y, dimension, mi_limits)
        binby = [binby] if isinstance(binby, str) else list(binby)
        if len(binby) > 3:
            raise ValueError("binby with dim > 3 is not yet supported")
        binby = [str(b) for b in binby]
        binby_shape = _expand_shape(shape, len(binby))
        combinations_unique, unique_reverse = _mi.unique_combinations(combinations)
        names = list(dict.fromkeys([str(e) for c in combinations_unique for e in c] + binby))
        f = self._with_columns(names)
        for e in names:
            if e in f.categories or _lib.dtype_of(f.columns[e]).kind in "mMO":
                raise NotImplementedError(f"mutual_information over the categorical, datetime or string column {e!r} is not supported")
        # the limits come from all rows of the frame, not the selection's (:762, :769), and every name's minmax once per call
        memo = {}
        binby_limits = f._limits_list(binby, limits, None, memo)
        values = _per_expression(mi_limits, len(combinations_unique))
        combination_limits = [f._limits_list([str(e) for e in c], v, None, memo) for c, v in zip(combinations_unique, values)]
        mask = f._selection(selection)
        dtypes = f.dtypes()
        plans = []
        for c, lims in zip(combinations_unique, combination_limits):
            c = [str(e) for e in c]
            specs = [_scalar_spec(e, dtypes[e], n, lim) for e, n, lim in zip(c, _expand_shape(mi_shape, len(c)), lims)]
            specs += [_scalar_spec(b, dtypes[b], n, lim) for b, n, lim in zip(binby, binby_shape, binby_limits)]
            plans.append((len(c), specs, 8 * int(np.prod([s["count"] + 3 for s in specs], dtype=np.int64))))
        budget, free = _mi.grid_budget(_lib.context().device)
        for (_, specs, nbytes), c in zip(plans, combinations_unique):
            if nbytes > free:
                shape_ = tuple(s["count"] for s in specs)
                raise MemoryError(f"mutual_information of {c}: the count grid of shape {shape_} (with edges, {nbytes} bytes) exceeds the "
                                  f"{free} bytes free on the device")
        mi_list = []
        for batch in _mi.batches([p[2] for p in plans], budget):
            tasks = []
            for i in batch:
                d, specs, _ = plans[i]
                part = taskpart.TaskPartCountGrid("mutual_information", specs, mask is not None, dtypes, _mi.finish, (d,), f.executor.nthreads)
                tasks.append(execution.Task(part, [mask]))
            f.executor.execute(f.columns, tasks, f.length, filter=f._filter)
            mi_list += [t.result for t in tasks]
            del tasks, part  # the batch's count grids go back before the next batch allocates
        return _mi.assemble(mi_list, x, unique_reverse, binby_shape, shape_result, waslist, sort)

    # ---- mode: the legacy histogram counted on the device, the argmax finish on the device (csrc/statistic.cu) ---------------
    def mode(self, expression, binby=[], limits=None, shape=256, mode_shape=64, mode_limits=None, selection=None):
        """df.mode (vaex/dataframe.py:2006-2034): per cell of the binby grid the center of the `mode_shape`-bin histogram bin of
        `expression` that holds the most rows (the first such bin), NaN where the cell is empty.  The histogram is vaex's legacy one
        (vaexfast histogram2d / 3d / Nd with their own bin rules, DESIGN.md section 3): the result is indexed with the LAST binby
        first, and with three binby every size must equal `mode_shape`.  `limits` / `mode_limits` are pairs, "minmax" / None or
        "N%"; `selection` is a boolean expression whose rows are counted.  A string `binby` is one expression."""
        from . import mode as _mode
        binby = [str(b) for b in ([binby] if isinstance(binby, str) else list(binby))]
        expression = str(expression)
        shape = _mode.grid_shape(binby, shape, mode_shape)
        names = list(dict.fromkeys(binby + [expression]))
        f = self._with_columns(names)
        for e in names:
            if _lib.dtype_of(f.columns[e]).kind not in "biuf":
                raise NotImplementedError(f"mode over the string, object or datetime column {e!r} is not supported")
        limits = list(f.limits(binby, limits)) + list(f.limits([expression], mode_limits))
        centers = _mode.centers(*limits[-1], mode_shape)
        _mode.check_memory(shape, _lib.context().device)
        mask = f._selection(selection)
        order = _mode.axis_order(binby + [expression])
        lims = _mode.axis_order(limits)
        part = taskpart.TaskPartMode(None, shape, order, [float(lim[0]) for lim in lims], [float(lim[1]) for lim in lims], centers,
                                     selection=mask is not None)
        task = execution.Task(part, [mask])
        f.executor.execute(f.columns, [task], f.length, filter=f._filter)
        return task.result

    # ---- binned statistics -------------------------------------------------------------------------------------------
    def _binner_specs(self, binby, limits, shape):
        binby, shapes, limits = _binned_args(binby, shape, limits)
        specs = []
        for i, b in enumerate(binby):
            if isinstance(b, dict):  # explicit spec (ordinal / hash binners)
                specs.append(b)
                continue
            dtype = _lib.dtype_of(self.columns[b])
            if b in self.categories:
                lo, count = self.categories[b]
                specs.append({"binner-type": "ordinal", "expression": b, "dtype": dtype.str, "count": count, "minimum": lo, "invert": False})
                continue
            lim = limits[i]
            if lim is None:
                lim = self.minmax(b).astype("float64")  # the extra pass the reference runs for limits=None (dataframe.py:5618)
            specs.append(_scalar_spec(b, dtype, shapes[i], lim))
        return specs

    def _agg(self, aggregators, binby=None, limits=None, shape=128, selection=None, edges=False, progress=None):
        """Run several aggregators in as few passes as possible (equal binners -> one fused pass); returns their results."""
        # a binby expression that is not a column (e.g. str_len(name)) is binned as a device-evaluated column
        f = self._with_columns([b for b in _binned_args(binby, shape, limits)[0] if isinstance(b, str)])
        if f is not self:
            return f._agg(aggregators, binby, limits, shape, selection, edges, progress)
        single = not isinstance(aggregators, (list, tuple))
        aggregators = [aggregators] if single else list(aggregators)
        specs = self._binner_specs(binby, limits, shape)
        dtypes = self.dtypes()
        # a LIST of selections gives one grid per selection, stacked along a new first axis (vaex/cpu.py:744-786, :798-811)
        selection = self._selection(selection)
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

    def skew(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.skew(self._as_float64(expression)), binby, limits, shape, selection, edges)

    def kurtosis(self, expression, binby=None, limits=None, shape=128, selection=None, edges=False):
        return self._agg(_agg.kurtosis(self._as_float64(expression)), binby, limits, shape, selection, edges)

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
        if _lib.dtype_of(col).kind == "f":
            return expression  # float32 already accumulates in double: identical result without the cast
        name = f"astype({expression}, 'float64')"
        if _lib.is_device(col):
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
        dt = _lib.dtype_of(col)
        counter = getattr(superutils, "counter_" + np.dtype(dt).newbyteorder("=").name)(1)
        chunk = self.executor.chunk_size_for(self.length) if not _lib.is_device(col) else max(self.length, 1)
        for i1 in range(0, self.length, chunk):
            data, mask = _lib.split_mask(col[i1:i1 + chunk])
            if mask is not None:
                counter.update(data, mask)
            else:
                counter.update(data if _lib.is_device(data) else np.ascontiguousarray(data))
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

    # ---- join: the right's index, the left's lookup and the row gathers on the device (vaex_b200/join.py) ----------------------
    def _index(self, expression, prime_growth=False, cardinality=None):
        """df._index (vaex/dataframe.py:514-572): the device index_hash_<T> of `expression` over the frame's rows"""
        from . import join as _join
        return _join.index(self, str(expression))

    def join(self, other, on=None, left_on=None, right_on=None, lprefix='', rprefix='', lsuffix='', rsuffix='', how='left', allow_duplication=False,
             prime_growth=False, cardinality_other=None, inplace=False):
        """df.join (vaex/join.py:125-297): `other`'s columns added to this frame's rows by the key `on` (or `left_on` / `right_on`:
        columns or expressions of numeric or datetime dtype), or side by side without a key.  how = 'left', 'right' or 'inner'; a
        right side with duplicate keys raises unless allow_duplication=True, and then repeats the left's rows, appended in (left row,
        right row) order.  The gathered columns land where the left key lives (torch on the device, numpy on the host; strings as
        arrow); a column with a missing row is a host np.ma array.  `prime_growth` and `cardinality_other` are ignored."""
        from . import join as _join
        return _join.join(self, other, on=on, left_on=left_on, right_on=right_on, lprefix=lprefix, rprefix=rprefix, lsuffix=lsuffix, rsuffix=rsuffix,
                          how=how, allow_duplication=allow_duplication, prime_growth=prime_growth, cardinality_other=cardinality_other, inplace=inplace)

    # ---- sort and take: the argsort and the row gathers on the device (vaex_b200/sort.py) --------------------------------------
    def take(self, indices, filtered=True, dropfilter=True):
        """df.take (vaex/dataframe.py:4444-4481): a frame of the rows `indices` (a list, numpy array or device tensor of integers),
        every real column gathered on the device (join's placement rule: device columns stay on the device, host ones come back to
        the host, strings as arrow, masks kept) and the virtual columns kept virtual.  With `filtered` the indices count the rows that
        pass this frame's filter; `dropfilter=False` keeps the filter over the taken rows.  An index outside [0, n) raises IndexError
        (the reference's numpy indexing would wrap a negative one)."""
        from . import sort as _sort
        return self._taken(_sort.take_index(self, indices, filtered), dropfilter)

    def sort(self, by, ascending=True):
        """df.sort (vaex/dataframe.py:4694-4745): the filtered rows ordered by `by` (a name, an expression or a list of them) as
        pa.compute.sort_indices orders them: stable, NaN after every number and null after NaN in either direction, strings bytewise.
        `ascending` is a bool or a list of them (a key ascends only when its flag `is True`, as there).  The result has no filter;
        a frame without rows that pass gives a copy of itself."""
        from . import sort as _sort
        by, ascending = _sort.normalize(by, ascending)
        rows = _sort.sorted_rows(self, by, ascending)
        if rows is None:
            return self._derive(self.columns)
        return self._taken(rows, True)

    def _taken(self, index, dropfilter):
        """a frame of the unfiltered rows `index`: real columns gathered, virtual ones over them, the filter dropped or kept"""
        from . import expression as _expr
        from . import join as _join
        real = {k: v for k, v in self.columns.items() if not isinstance(v, _expr.DeviceExpression)}
        out = self._derive(_join.gather(real, index, self.length, _lib.is_device), drop_filter=True)
        for name, col in self.columns.items():
            if isinstance(col, _expr.DeviceExpression):
                out.add_virtual_column(name, col.expression)
        out.columns = {name: out.columns[name] for name in self.columns}  # the column order of this frame
        if not dropfilter and self._filter_expression is not None:
            out = out.filter(self._filter_expression)
        return out

    # ---- groupby ------------------------------------------------------------------------------------------------------
    def groupby(self, by, agg=None, sort=False, fused=True, combine=False):
        """df.groupby(by).agg(agg): `by` is a name, an expression, a binner (Binner, BinnerInteger, BinnerTime) or a list mixing them;
        one output row per group with rows"""
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
        self.by = [by] if isinstance(by, (str, BinnerBase)) else list(by)
        binners = [b for b in self.by if isinstance(b, BinnerBase)]
        df = df._with_columns([b.expression if isinstance(b, BinnerBase) else b for b in self.by])  # a key that is an expression: a virtual column
        self.df = df
        self.fused = fused
        self.sort = sort
        self.combined = None
        self.hash_maps = []
        for name in self.by:
            if isinstance(name, BinnerBase):
                continue
            col = df.columns[name]
            part = taskpart.TaskPartHashmapUniqueCreate(None, name, _lib.dtype_of(col), nthreads=1)
            # nthreads=1 -> 7 shards, chunks fed in row order: the ordinals of the sequential reference run
            task = execution.Task(part)
            ex = execution.Executor(1, chunk_size_max=df.executor.chunk_size_max)
            ex.execute(df.columns, [task], df.length, filter=df._filter)
            hm = task.result
            if sort:
                hm = hm.sorted()
            self.hash_maps.append(hm)
        if binners:
            # a binner's cells are fixed before the pass: the grid stays dense under combine="auto"
            if combine is True and len(self.by) >= 2:
                raise NotImplementedError(f"cannot combine {binners[0]!r} with other groupers: the sparse combine path takes hashed keys only")
            return
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
        return [k.bin_values if isinstance(k, BinnerBase) else hm.keys() for k, hm in zip(self.by, self._key_maps())]

    def _key_maps(self):
        """the hash map of every hashed key, None for a binner, in the order of `by`"""
        maps = iter(self.hash_maps)
        return [None if isinstance(k, BinnerBase) else next(maps) for k in self.by]

    def agg(self, actions):
        """actions: {column: [names]} | {column: name} | [descriptors]; returns dict of arrays (one row per non-empty group)."""
        df = self.df
        descs, labels = [], []
        columns = dict(df.columns)
        if isinstance(actions, str):  # df.groupby(by, agg='count') (vaex/groupby.py:688-700)
            by = [k.expression if isinstance(k, BinnerBase) else k for k in self.by]
            actions = [_agg.aggregates[actions]("*")] if actions == "count" else {c: actions for c in df.columns if c not in by}
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
            frame = df._derive(columns)
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
        # per key: its label, the cells of its grid axis, the first cell of a group and the group keys
        axes = []
        for name, hm in zip(self.by, self._key_maps()):
            if hm is None:  # a binner: its cells are fixed (vaex_b200/groupby.py)
                specs.append(name.spec(df))
                axes.append((name.label, name.cells, name.start, name.bin_values))
                continue
            axes.append((name, len(hm) + 2, 0, hm.keys()))
            dtype = _lib.dtype_of(df.columns[name])
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
                cdt = _lib.dtype_of(codes)
                specs.append({"binner-type": "ordinal", "expression": cname, "dtype": cdt.str, "count": len(hm), "minimum": 0, "invert": False})
        frame = df._derive(columns)
        grids = frame._agg(descs, binby=specs, edges=True)
        # _extract_center (vaex/groupby.py:896-977): drop the null / nan edge cells, keep groups with count > 0
        center = tuple(slice(start, start + len(keys)) for _, _, start, keys in axes)
        counts = grids[-1][center]
        keep = counts > 0
        out = {}
        mesh = np.meshgrid(*[np.arange(len(keys)) for _, _, _, keys in axes], indexing="ij")
        for (label, _, _, keys), m in zip(axes, mesh):
            out[label] = keys[m[keep]]
        # a list aggregator returns ONE arrow list per cell of the flat FULL grid (first binner fastest, edge cells included)
        shape = [cells for _, cells, _, _ in axes]
        strides = np.cumprod([1] + shape[:-1])
        flat = sum((i.astype(np.int64) + start) * int(st) for i, st, (_, _, start, _) in zip(np.nonzero(keep), strides, axes))
        for label, g in zip(labels[:-1], grids[:-1]):
            out[label] = _take_cells(g, flat) if _is_arrow(g) else g[center][keep]
        out["count"] = counts[keep]
        return out


def _boolean_selection(mask):
    """a resolved selection argument, checked to be boolean"""
    if mask.dtype != np.bool_:
        raise ValueError("a selection must be a boolean expression")
    return mask


def _issequence(x):
    return isinstance(x, (tuple, list, np.ndarray))


def _per_expression(value, n):
    """df.limits' broadcast: one limit value (a pair, a string or None) for all n expressions, else one per expression"""
    return (value,) * n if _is_limit(value) or not _issequence(value) else value


def _is_limit(x):
    """vaex.utils._is_limit: a sequence of numbers"""
    import numbers
    return _issequence(x) and all(isinstance(k, numbers.Number) for k in x)


def _expand_shape(shape, dimension):
    """vaex.utils._expand_shape"""
    if isinstance(shape, (tuple, list)):
        assert len(shape) == dimension, "wants to expand shape %r to dimension %d" % (shape, dimension)
        return tuple(shape)
    return (shape,) * dimension


def _expand_limits(limits, dimension):
    """vaex.utils._expand_limits"""
    if _issequence(limits) and (_issequence(limits[0]) or isinstance(limits[0], str) or limits[0] is None):
        assert len(limits) == dimension, "wants to expand shape %r to dimension %d" % (limits, dimension)
        return tuple(limits)
    return (limits,) * dimension


def _minmax_as(res, dtype):
    """the (min, max) doubles cast back to the column's dtype (vaex/dataframe.py:1524-1528); datetimes stay raw doubles"""
    dt = np.dtype(dtype).newbyteorder("=")
    if dt.kind in "mM":
        return res
    with np.errstate(invalid="ignore"):
        return res.astype(dt)


def _binned_args(binby, shape, limits):
    """binby, shape and limits of the binned and legacy statistics -> (binby list, one shape per binby, one limit pair or None per
    binby); None or a string `limits` (whatever it says) leaves every limit to the minmax pass"""
    binby = [] if binby is None else [binby] if isinstance(binby, (str, dict)) else list(binby)
    shapes = [shape] * len(binby) if np.isscalar(shape) else list(shape)
    limits = [None] * len(binby) if limits is None or isinstance(limits, str) else list(limits)
    if len(binby) == 1 and len(limits) == 2 and np.isscalar(limits[0]):
        limits = [limits]
    return binby, shapes, limits


def _scalar_spec(expression, dtype, count, limit):
    """the spec of a BinnerScalar (vaex/dataframe.py:7294-7360)"""
    return {"binner-type": "scalar", "expression": expression, "dtype": dtype.str, "count": int(count), "minimum": float(limit[0]),
            "maximum": float(limit[1])}


def _is_arrow(x):
    return type(x).__module__.startswith("pyarrow")


def _take_cells(lists, cells):
    import pyarrow as pa
    return lists.take(pa.array(np.asarray(cells, dtype=np.int64)))
