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


def _issequence(x):
    return isinstance(x, (tuple, list))


def _is_device(x):
    return hasattr(x, "__cuda_array_interface__") and not isinstance(x, np.ndarray)


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
        N = i2 - i1
        if filter_mask is not None:  # the executor compacted the blocks with the filter (vaex/execution.py:516-522)
            kept = getattr(filter_mask, "kept", None)
            N = len(blocks[0]) if blocks else (int(kept) if kept is not None else int(np.asarray(filter_mask).sum()))
        for block in blocks:
            assert len(block) == N, f"Oops, got a block of length {len(block)} while it is expected to be of length {N} (at {i1}-{i2}, filter={filter_mask is not None})"
        block_map = {expr: block for expr, block in zip(self.expressions, blocks)}

        def split(block):
            """-> (data, numpy-style mask or None); datetimes travel as integers (vaex/cpu.py:692-694)."""
            if _is_device(block) or _hash.is_string_column(block):
                return block, None  # string columns go to AggCount_string / AggNUnique_string as they are
            if np.ma.isMaskedArray(block):
                return np.ascontiguousarray(block.data), np.ma.getmaskarray(block)
            block = np.asarray(block)
            if block.dtype.kind in "mM":
                block = block.view("uint64")
            return block, None

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
                    if not _is_device(selection_mask):
                        selection_mask = np.asarray(selection_mask)
                        if np.ma.isMaskedArray(selection_mask):  # vaex.utils.unmask_selection_mask
                            selection_mask = selection_mask.data & ~np.ma.getmaskarray(selection_mask)
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
        N = i2 - i1
        if filter_mask is not None:  # the executor compacted the blocks with the filter
            kept = getattr(filter_mask, "kept", None)
            N = len(blocks[0]) if blocks else (int(kept) if kept is not None else int(np.asarray(filter_mask).sum()))
        nd = len(self.expressions)
        if not blocks and self.op.code != _stat.OP_ADD1.code:
            raise ValueError("Nothing to compute for OP %s" % self.op.code)
        for block in blocks[nd:]:
            if _hash.is_string_column(block) or (not _is_device(block) and np.asarray(block).dtype.kind not in "biufmM"):
                raise NotImplementedError("the legacy statistic of a string or object column has no GPU path")
        dtypes = [np.dtype(block.__cuda_array_interface__["typestr"]) if _is_device(block) else block.dtype for block in blocks]
        cls = _stat.compute_class(dtypes) if dtypes else _lib.F32
        sels = []
        for i, selection in enumerate(self.selections):
            if selection is None or selection is False:
                sels.append(None)
                continue
            mask = selection_masks[i]
            if mask is None:
                raise ValueError("performing operation on selection while no selection present")
            if not _is_device(mask):
                mask = np.asarray(mask.data & ~np.ma.getmaskarray(mask)) if np.ma.isMaskedArray(mask) else np.asarray(mask)  # unmask_selection_mask
            sels.append(mask)
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


REGISTRY = {cls.snake_name: cls for cls in (TaskPartAggregation, TaskPartHashmapUniqueCreate)}


def install_into_vaex():
    """Register the GPU task parts under vaex's 'task-part-cpu' registry names so ExecutorLocal picks them up
    (vaex/cpu.py:21, vaex/execution.py:385-399).  See INTEGRATION.md; needs an importable vaex."""
    import vaex.cpu  # noqa: F401  (not importable in the build container: dask/frozendict/aplus/future missing)
    from . import vaex_plugin
    return vaex_plugin.install()
