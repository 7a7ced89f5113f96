"""Task parts — the drop-in boundary B1 of SURVEY.md section 8b.

``TaskPartAggregation`` and ``TaskPartHashmapUniqueCreate`` keep the interface the reference executor drives
(packages/vaex-core/vaex/cpu.py:629-845 and :285-405; called from vaex/execution.py:385-412, :564, :451-453):

    decode(encoding, spec, df, nthreads) / process(thread_index, i1, i2, filter_mask, selection_masks, blocks) /
    reduce(others) / get_result() / ideal_splits(nthreads) / memory_usage() / get_bin_count() / .stopped / .expressions

The spec dicts are the ones vaex's tasks encode (vaex/tasks.py:498-504, vaex/dataframe.py:7294-7360, vaex/agg.py:240-252).
``blocks`` may be numpy / numpy.ma arrays (host chunks: staged to the device per call on the slot of ``thread_index``) or
device arrays (``__cuda_array_interface__``; zero copy).  All per-row work happens in libb200agg.so.
"""
import sys
from functools import reduce

import numpy as np

from . import _lib
from . import agg as _agg
from . import hash as _hash
from . import superagg
from . import superutils


def _issequence(x):
    return isinstance(x, (tuple, list))


def _rows(i1, i2, filter_mask, blocks):
    """the rows of a chunk the part sees: all of [i1, i2), or those the filter kept when the executor compacted the blocks with it
    (vaex/execution.py:516-522); count(*) has no block to take that length from"""
    if filter_mask is None:
        return i2 - i1
    kept = getattr(filter_mask, "kept", None)
    return len(blocks[0]) if blocks else (int(kept) if kept is not None else int(np.asarray(filter_mask).sum()))


def decode_binner(spec, nthreads, hash_maps=None):
    """binner_encoding.decode (vaex/cpu.py:46-65)."""
    kind = spec.get("binner-type", spec.get("type"))
    dtype = np.dtype(spec["dtype"])
    if kind == "ordinal":
        cls = _agg.find_type_from_dtype(superagg, "BinnerOrdinal_", dtype)
        return cls(nthreads, spec["expression"], spec["count"], spec["minimum"], False, spec.get("invert", False))
    if kind == "scalar":
        cls = _agg.find_type_from_dtype(superagg, "BinnerScalar_", dtype)
        return cls(nthreads, spec["expression"], spec["minimum"], spec["maximum"], spec["count"])
    if kind == "hash":
        cls = _agg.find_type_from_dtype(superagg, "BinnerHash_", dtype)
        hm = spec["hash_map_unique"]
        if not isinstance(hm, _hash.HashMapUnique):
            hm = (hash_maps or {})[hm]
        return cls(nthreads, spec["expression"], hm)
    if kind == "time":  # a datetime64[unit] column (its ticks as int64) -> periods of `resolution` (vaex_b200/groupby.py BinnerTime)
        unit, step = np.datetime_data(dtype)
        if dtype.kind != "M" or step != 1:
            raise ValueError(f"a time binner needs a datetime64 column with a plain unit, not {dtype}")
        cls = _agg.find_type_from_dtype(superagg, "BinnerTime_", np.dtype("int64").newbyteorder(dtype.byteorder))
        return cls(nthreads, spec["expression"], unit, spec["resolution"], spec["begin"], spec["count"], spec.get("every", 1))
    raise ValueError("Cannot deserialize: %r" % spec)


class TaskPart:
    stopped = False

    def ideal_splits(self, nthreads):
        return nthreads

    def memory_usage(self):
        return 0


class TaskPartAggregation(TaskPart):
    """vaex/cpu.py:629-845."""
    snake_name = "aggregations"

    def __init__(self, df, binners, aggregation_descriptions, dtypes, initial_values=None, nthreads=None):
        self.df = df
        self.has_values = False
        self.dtypes = dtypes
        self.binners = binners
        self.nthreads = nthreads or 1
        self.expressions = [binner.expression for binner in binners]
        self.aggregation_descriptions = aggregation_descriptions
        for d in self.aggregation_descriptions:
            self.expressions.extend(d.expressions)
        self.grid = superagg.Grid([binner.copy() for binner in binners])
        self.nbytes = 0
        # vaex/agg.py:311-318 pre-declares bytes_per_cell * cells * grids per aggregator and cross-checks it against the object;
        # the executor compares the sum with memory_usage() (vaex/execution.py:413-414)
        self.predicted_memory_usage = 0
        self.aggregations = []
        for i, d in enumerate(self.aggregation_descriptions):
            selection = d.selection
            selection_waslist = _issequence(selection)
            selections = list(selection) if selection_waslist else [selection]
            ops = []
            for j, _ in enumerate(selections):
                op = d._create_operation(self.grid, self.nthreads)
                self.nbytes += sys.getsizeof(op)
                self.predicted_memory_usage += getattr(d, "predicted_memory_usage", sys.getsizeof(op))
                if initial_values is not None:
                    op.load(initial_values[i][j])  # vaex/cpu.py:654-658
                ops.append(op)
            self.aggregations.append((d, selections, ops, selection_waslist))

    def get_bin_count(self):
        return reduce(lambda prev, binner: len(binner) * prev, self.binners, 1)

    def memory_usage(self):
        return self.nbytes

    def ideal_splits(self, nthreads):
        return 1  # one part shared by every thread (vaex/cpu.py:675-676)

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        # vaex/cpu.py:678-786
        N = _rows(i1, i2, filter_mask, blocks)
        for block in blocks:
            assert len(block) == N, f"Oops, got a block of length {len(block)} while it is expected to be of length {N} (at {i1}-{i2}, filter={filter_mask is not None})"
        block_map = {expr: block for expr, block in zip(self.expressions, blocks)}

        def split(block):
            """-> (data, numpy-style mask or None); datetimes travel as integers (vaex/cpu.py:692-694)."""
            if _hash.is_string_column(block):
                return block, None  # string columns go to AggCount_string / AggNUnique_string as they are
            data, mask = _lib.split_mask(block)
            if not _lib.is_device(data):
                data = np.asarray(data)
                if data.dtype.kind in "mM":
                    data = data.view("uint64")
            return data, mask

        for binner in self.grid.binners:
            data, mask = split(block_map[binner.expression])
            binner.set_data(thread_index, data)
            if mask is not None:
                binner.set_data_mask(thread_index, mask)  # 1 = masked
            else:
                binner.clear_data_mask(thread_index)
        all_aggregators = []
        selection_index_global = 0
        for agg_desc, selections, ops, _ in self.aggregations:
            for selection_index, selection in enumerate(selections):
                op = ops[selection_index]
                all_aggregators.append(op)
                selection_mask = None
                if not (selection is None or selection is False):
                    selection_mask = selection_masks[selection_index_global]
                    assert selection_mask is not None
                    selection_mask = _lib.unmask_selection(selection_mask)
                    # some aggregators make a distinction between missing value and no value (nunique): vaex/cpu.py:750-756
                    if hasattr(op, "set_selection_mask"):
                        op.set_selection_mask(thread_index, selection_mask)
                elif hasattr(op, "clear_selection_mask"):
                    op.clear_selection_mask(thread_index)
                selection_index_global += 1
                for i, expression in enumerate(agg_desc.expressions):
                    data, mask = split(block_map[expression])
                    op.set_data(thread_index, data, i)
                    if mask is not None:
                        # one combined validity mask per aggregator: selection & ~mask, 1 = use the row (vaex/cpu.py:765-784)
                        selection_mask = ~mask if selection_mask is None else (np.asarray(selection_mask, bool) & ~mask)
                if selection_mask is not None:
                    op.set_data_mask(thread_index, selection_mask)
                else:
                    op.clear_data_mask(thread_index)
        self.grid.bin(thread_index, all_aggregators, N, row_offset=i1)
        self.has_values = True

    def reduce(self, others):
        for agg_index, (_, selections, ops, _) in enumerate(self.aggregations):
            for selection_index, _ in enumerate(selections):
                ops[selection_index].merge([o.aggregations[agg_index][2][selection_index] for o in others])

    def get_result(self):
        # vaex/cpu.py:798-811
        results = []
        for agg_desc, selections, ops, selection_waslist in self.aggregations:
            grids = [agg_desc.get_result(op) for op in ops]
            if type(grids[0]).__module__.startswith("pyarrow"):  # AggList: one arrow large_list per cell (immutable, nothing to copy)
                results.append(grids if selection_waslist else grids[0])
                continue
            result = np.asarray(grids) if selection_waslist else grids[0]
            if not np.ma.isMaskedArray(result):
                result = result.copy()
            results.append(result)
        return results

    def get_values(self):
        return [[np.asarray(op) for op in ops] for _, _, ops, _ in self.aggregations]

    @classmethod
    def decode(cls, encoding, spec, df=None, nthreads=1):
        """``spec`` = TaskAggregations.encode() (vaex/tasks.py:498-504).  ``encoding`` is only consulted for hash-map objects."""
        aggs = [_agg.from_spec(s) for s in spec["aggregations"]]
        dtypes = {k: np.dtype(v) for k, v in spec["dtypes"].items()}
        hash_maps = getattr(encoding, "hash_maps", None) if encoding is not None else None
        binners = [decode_binner(b, nthreads, hash_maps) for b in spec["binners"]]
        for a in aggs:
            a._prepare_types(dtypes)
        values = spec.get("values")
        return cls(df, binners, aggs, dtypes, initial_values=values, nthreads=nthreads)

    def encode(self, encoding=None):
        encoded = {"aggregations": [d.encode() for d in self.aggregation_descriptions], "dtypes": {k: str(v) for k, v in self.dtypes.items()}}
        if self.has_values:
            encoded["values"] = self.get_values()
        return encoded


class TaskPartCountGrid(TaskPartAggregation):
    """A count(*) pass with edges over `specs` on one device grid, then `finish(grid pointer, grid sizes, *args, ctx=...)` on that grid;
    only the finish's answer is read back, the count grid never leaves the device.  Two analyses run through it:
      * "percentile_approx": one expression of percentile_approx / median_approx (vaex/dataframe.py:1632-1780), binby + [expression]
        (:1668-1672), finished by percentile.finish with args (the expression's (lb, ub) limit, percentage) (csrc/percentile.cu);
      * "mutual_information": one combination of mutual_information (vaex/dataframe.py:685-819), combination + binby (:796-797),
        finished by mutual_information.finish with args (the number of leading MI axes,) (csrc/mutinfo.cu)."""

    def __init__(self, snake_name, specs, selection, dtypes, finish, args, nthreads=1):
        desc = _agg.count("*", selection="selection" if selection else None, edges=True)
        desc._prepare_types(dtypes)
        super().__init__(None, [decode_binner(s, nthreads) for s in specs], [desc], dtypes, nthreads=nthreads)
        self.snake_name = snake_name
        self.finish = finish
        self.args = tuple(args)

    def get_result(self):
        op = self.aggregations[0][2][0]
        if op.device_dtype != np.int64:
            raise RuntimeError(f"the {self.snake_name} finish reads an int64 count grid")
        ptr, _ = op.device_pointer(0)
        return self.finish(ptr, self.grid.shapes, *self.args, ctx=op._ctx)


class RowLimitException(ValueError):
    pass


class TaskPartHashmapUniqueCreate(TaskPart):
    """vaex/cpu.py:285-405 — pass 1 of a groupby: build the ordered set of keys."""
    snake_name = "hash_map_unique_create"

    def __init__(self, df, expression, dtype, dtype_item=None, flatten=False, limit=None, limit_raise=True, selection=None, nthreads=1,
                 return_inverse=False):
        self.df = df
        self.nthreads = nthreads
        self.dtype = np.dtype(dtype)
        self.dtype_item = np.dtype(dtype_item if dtype_item is not None else dtype)
        self.flatten = flatten
        self.expression = str(expression)
        self.limit = limit
        self.limit_raise = limit_raise
        self.selection = selection
        self.return_inverse = return_inverse
        self.chunks = []
        self.values = None
        self.fingerprint = ""
        # the reference uses nthreads*7 shards to dodge lock contention (vaex/cpu.py:317); kept so ordinals agree with it
        self.hash_map_unique = _hash.HashMapUnique(self.dtype_item, self.nthreads * 7, limit=self.limit)

    def get_bin_count(self):
        return len(self.hash_map_unique)

    @property
    def expressions(self):
        return [self.expression]

    def get_result(self):
        return (self.hash_map_unique, self.values) if self.return_inverse else self.hash_map_unique

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        ar = blocks[0]
        self._check_row_limit()
        if self.stopped:
            return
        if self.selection:
            m = np.asarray(selection_masks[0], bool)
            ar = ar[m]
        if len(ar) == 0:
            return
        result = self.hash_map_unique.add(ar, return_inverse=self.return_inverse)
        if self.return_inverse:
            values, map_index = result
            self.chunks.append((i1, i2, values, map_index))
        self._check_row_limit()

    def _check_row_limit(self):
        if self.limit is not None:
            if self.limit_raise and len(self.hash_map_unique) > self.limit:
                raise RowLimitException(f"Resulting hash_map_unique would have >= {self.limit} unique combinations")
            if not self.limit_raise and len(self.hash_map_unique) >= self.limit:
                self.stopped = True

    def ideal_splits(self, nthreads):
        return 1

    def reduce(self, others):
        merged = self.hash_map_unique
        if others:
            merged.merge([o.hash_map_unique for o in others if o.hash_map_unique is not None])
        if self.return_inverse:
            self.chunks.sort(key=lambda x: x[0])
            length = sum(len(c[2]) for c in self.chunks)
            self.values = np.empty(length, np.int64)
            for i1, i2, values, map_index in self.chunks:
                merged._internal.flatten_values(values, map_index, self.values[i1:i2])
        if self.limit is not None:
            count = len(merged)
            if count > self.limit:
                if self.limit_raise:
                    raise RowLimitException(f"Resulting set has {count:,} unique combinations, which is larger than the allowed value of {self.limit:,}")
                merged = merged.limit(self.limit)
        self.hash_map_unique = merged.flatten()
        self.hash_map_unique._internal.fingerprint = f"hash-map-unique-{self.fingerprint}"

    @classmethod
    def decode(cls, encoding, spec, df=None, nthreads=1):
        return cls(df, spec["expression"], spec["dtype"], spec.get("dtype_item", spec["dtype"]), flatten=spec.get("flatten", False), limit=spec.get("limit"),
                   limit_raise=spec.get("limit_raise", True), selection=spec.get("selection"), return_inverse=spec.get("return_inverse", False),
                   nthreads=nthreads)

    def memory_usage(self):
        return self.hash_map_unique._internal.__sizeof__()


def _key_block(block):
    """a join key block -> (keys, mask or None): datetimes and timedeltas travel as int64 (vaex/join.py:192-193)"""
    block, mask = _lib.split_mask(block)
    if _lib.is_device(block):
        return block, None
    block = np.asarray(block)
    return (block.view(np.int64) if block.dtype.kind in "mM" else block), mask


class TaskPartIndex(TaskPart):
    """DataFrame._index (vaex/dataframe.py:514-572): ONE device index_hash_<T> for the pass; every thread updates it on its own slot
    with its chunk's global rows.  The index follows the sequential rule whatever the thread count and chunk order, so the reference's
    per-thread indices and their merge (:540-571) have nothing to do here."""

    def __init__(self, expression, dtype, nmaps=1):
        self.expression = str(expression)
        self.expressions = [self.expression]
        self.index = _hash.index_type_from_dtype(dtype)(nmaps)
        self._ctx = _lib.context()

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        assert filter_mask is None, "the indexed side of a join is extracted first: its rows are its unfiltered rows"
        keys, mask = _key_block(blocks[0])
        self.index.update(keys, masks=mask, start_index=i1, slot=self._ctx.slot(thread_index))

    def reduce(self, others):
        pass

    def get_result(self):
        return self.index


class TaskPartLookup(TaskPart):
    """The lookup pass of vaex/join.py:185-209 over every unfiltered row of the left key (run without the filter): map_index /
    map_index_masked into `lookup[i1:i2]` (host or device), and with duplicates on the right map_index_duplicates, kept on the
    device.  Result: (whether a row found nothing, [(i1, left rows, right rows)] in row order)."""

    def __init__(self, index, expression, lookup, duplicates):
        import threading
        self.index = index
        self.expression = str(expression)
        self.expressions = [self.expression]
        self.lookup = lookup
        self.duplicates = duplicates
        self.unknown = False
        self.extra = []
        self._lock = threading.Lock()
        self._ctx = _lib.context()

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        keys, mask = _key_block(blocks[0])
        native = self.index._np_dtype()
        slot = self._ctx.slot(thread_index)
        if _lib.is_device(keys) and _lib.dtype_of(keys) != native:
            keys = superutils.device_cast(keys, native, self._ctx)  # once for map_index and map_index_duplicates
        out = self.lookup[i1:i2]
        if mask is None:
            unknown = self.index.map_index(keys, out, slot=slot)
        else:
            unknown = self.index.map_index_masked(keys, mask, out, slot=slot)
        extra = self.index.map_index_duplicates(keys, i1, mask, device=True, slot=slot) if self.duplicates else None
        with self._lock:
            self.unknown = self.unknown or bool(unknown)
            if extra is not None and len(extra[0]):
                self.extra.append((i1,) + tuple(extra))

    def reduce(self, others):
        self.extra.sort(key=lambda e: e[0])

    def get_result(self):
        return self.unknown, self.extra


class TaskPartStatistic(TaskPart):
    """vaex/cpu.py:487-626 — the legacy statistics (df.cov, df.correlation, binned df.minmax, the limits pre-pass) on one device
    grid per compute class (csrc/statistic.cu).  ``blocks`` are the binby blocks followed by the weight blocks."""
    snake_name = "legacy_statistic"

    def __init__(self, df, shape, expressions, dtype, selections, op, weights, minima, maxima, edges, selection_waslist):
        self.df = df
        self.shape = tuple(shape)
        self.dtype = dtype
        self.expressions = list(expressions)
        self.op = op
        self.weights = list(weights)
        self.selections = list(selections)
        self.fields = op.fields(weights)
        self.shape_total = (len(self.selections),) + self.shape + (self.fields,)
        self.minima = list(minima)
        self.maxima = list(maxima)
        self.edges = edges
        self.selection_waslist = selection_waslist
        self.stats = {}  # compute class -> _stat.Statistic, created on the first chunk of that class
        self.grid = None

    def get_bin_count(self):
        return reduce(lambda a, b: a * b, self.shape, 1)

    def ideal_splits(self, nthreads):
        return 1  # one device grid shared by every thread

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        from . import statistic as _stat
        N = _rows(i1, i2, filter_mask, blocks)
        nd = len(self.expressions)
        if not blocks and self.op.code != _stat.OP_ADD1.code:
            raise ValueError("Nothing to compute for OP %s" % self.op.code)
        for block in blocks[nd:]:
            if _hash.is_string_column(block) or (not _lib.is_device(block) and np.asarray(block).dtype.kind not in "biufmM"):
                raise NotImplementedError("the legacy statistic of a string or object column has no GPU path")
        dtypes = [_lib.dtype_of(block) for block in blocks]
        cls = _stat.compute_class(dtypes) if dtypes else _lib.F32
        sels = []
        for i, selection in enumerate(self.selections):
            if selection is None or selection is False:
                sels.append(None)
                continue
            mask = selection_masks[i]
            if mask is None:
                raise ValueError("performing operation on selection while no selection present")
            sels.append(_lib.unmask_selection(mask))
        stat = self.stats.get(cls)
        if stat is None:
            stat = self.stats.setdefault(cls, _stat.Statistic(self.op.code, cls, self.shape, self.minima, self.maxima, self.edges,
                                                              len(self.weights), len(self.selections)))
        stat.bin(thread_index, blocks[:nd], blocks[nd:], sels, N, row_offset=i1)
        return i2 - i1

    def _grids(self):
        if not self.stats:
            grid = np.zeros(self.shape_total, np.float64)
            self.op.init(grid)
            return [grid]
        return [s.read() for s in self.stats.values()]

    def reduce(self, others):
        # vaex/cpu.py:613-616: the op's own reduce over every grid (nansum / sum / nanmin+nanmax / argmin of the order)
        grids = self._grids() + [g for o in others for g in o._grids()]
        dtype = np.dtype(getattr(self.dtype, "numpy", self.dtype))
        self.grid = self.op.reduce(np.array(grids).astype(dtype, copy=False))
        for s in self.stats.values():
            s.close()
        self.stats = {}

    def get_result(self):
        if self.grid is None:
            self.reduce([])
        return self.grid if self.selection_waslist else self.grid[0]

    @classmethod
    def decode(cls, encoding, spec, df=None, nthreads=1):
        """``spec`` = TaskStatistic.encode() (vaex/tasks.py:409-413); without an ``encoding`` the '_op' spec is decoded locally"""
        from . import statistic as _stat
        spec = dict(spec)
        if encoding is not None:
            spec["op"] = encoding.decode("_op", spec["op"])
            spec["dtype"] = encoding.decode("dtype", spec["dtype"])
        elif isinstance(spec["op"], dict):
            spec["op"] = _stat.decode_op(spec["op"])
        return cls(df, **spec)


class TaskPartMode(TaskPart):
    """df.mode (vaex/dataframe.py:2006-2034): vaex.legacy.TaskHistogram's count of binby + [expression] (vaex/legacy.py:22-110) on one
    device histogram (csrc/statistic.cu, b200_stat_create_histogram), then the argmax finish on that grid; only the modes are read
    back.  ``expressions`` are in grid axis order, the reference's blocks reversed (mode.axis_order); ``shape``, ``minima`` and
    ``maxima`` follow them.  Values are binned as float64 (``_asfloat``), masked columns by the values under their mask, as vaexfast
    reads them; ``selection`` = the task's first selection mask compacts the rows, like a filter does."""
    snake_name = "mode"

    def __init__(self, df, shape, expressions, minima, maxima, centers, selection=False):
        from . import mode as _mode
        self.df = df
        self.shape = tuple(int(s) for s in shape)
        self.expressions = list(expressions)
        self.centers = centers
        self.selection = bool(selection)
        self.histogram = _mode.Histogram(self.shape, minima, maxima)
        self.result = None

    def get_bin_count(self):
        return reduce(lambda a, b: a * b, self.shape, 1)

    def ideal_splits(self, nthreads):
        return 1  # one device grid shared by every thread

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        N = len(blocks[0])
        columns = []
        for block in blocks:
            if _hash.is_string_column(block) or (not _lib.is_device(block) and np.asarray(block).dtype.kind not in "biuf"):
                raise NotImplementedError("mode of a string, object or datetime column has no GPU path")
            columns.append(_lib.split_mask(block)[0])
        selection = _lib.unmask_selection(selection_masks[0]) if self.selection else None
        self.histogram.bin(thread_index, columns, [], [selection], N, row_offset=i1)
        return i2 - i1

    def reduce(self, others):
        if others:
            raise ValueError("a mode task part is never split")
        if self.result is None:
            self.result = self.histogram.mode(self.centers)
            self.histogram.close()

    def get_result(self):
        self.reduce([])
        return self.result


REGISTRY = {cls.snake_name: cls for cls in (TaskPartAggregation, TaskPartHashmapUniqueCreate)}


def install_into_vaex():
    """Register the GPU task parts under vaex's 'task-part-cpu' registry names so ExecutorLocal picks them up
    (vaex/cpu.py:21, vaex/execution.py:385-399).  See INTEGRATION.md; needs an importable vaex."""
    import vaex.cpu  # noqa: F401  (not importable in the build container: dask/frozendict/aplus/future missing)
    from . import vaex_plugin
    return vaex_plugin.install()
