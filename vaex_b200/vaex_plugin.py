"""Registration of the GPU task parts inside a real vaex installation (boundary B1).

``import vaex`` fails in the build container (dask / frozendict / aplus / future are missing and there is no network), so this
module is written against the interface in /root/reference and EXERCISED through a stub ``vaex`` package that restates exactly the
pieces it touches — the 'task-part-cpu' class registry (vaex/encoding.py:31-52), ``encoding.decode``, ``vaex.memory.local.agg`` and
``vaex.array_types.to_numpy`` — in tests/test_gpu_vaex_plugin_stub.py: the spec dicts ``TaskAggregations.encode`` emits
(vaex/tasks.py:498-504) are decoded into the GPU task parts through the registry and driven like ExecutorLocal does.
INTEGRATION.md walks through it.

How vaex finds task parts: ``vaex.cpu.register = vaex.encoding.make_class_registery('task-part-cpu')``
(packages/vaex-core/vaex/cpu.py:21, vaex/encoding.py:31-52) keeps a dict ``snake_name -> class``; ExecutorLocal renames the
task spec's ``task-type`` to ``task-part-cpu-type`` and calls ``encoding.decode('task-part-cpu', spec, df=, nthreads=)``
(vaex/execution.py:385-399).  Registering a class with the same ``snake_name`` ("aggregations",
"hash_map_unique_create") replaces the CPU implementation for every DataFrameLocal in the process.
"""
import numpy as np

from . import agg as _agg
from . import taskpart as _tp


def _np_dtype(encoding, spec_dtype):
    dt = encoding.decode("dtype", spec_dtype)
    return np.dtype(getattr(dt, "numpy", dt))


class VaexTaskPartAggregation(_tp.TaskPartAggregation):
    snake_name = "aggregations"

    @classmethod
    def decode(cls, encoding, spec, df, nthreads):
        import vaex.memory
        dtypes = {k: _np_dtype(encoding, v) for k, v in spec["dtypes"].items()}
        binners = []
        for b in spec["binners"]:
            b = dict(b)
            b["dtype"] = _np_dtype(encoding, b["dtype"]).str
            if b.get("binner-type") == "hash":
                hid = b["hash_map_unique"]
                raise NotImplementedError(f"hash binner {hid}: vaex keeps _EXPERIMENTAL_BINNER_HASH off (vaex/groupby.py:28); groupby arrives as ordinal binners")
            binners.append(_tp.decode_binner(b, nthreads))
        aggs = [_agg.from_spec(s) for s in spec["aggregations"]]
        for a in aggs:
            a._prepare_types(dtypes)
        part = cls(df, binners, aggs, dtypes, nthreads=nthreads)
        # keep the executor's accounting consistent (vaex/execution.py:413-414): declare what the device grids hold
        vaex.memory.local.agg.pre_alloc(part.memory_usage(), "GPU aggregator grids (device)")
        return part

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        import vaex.array_types
        from . import hash as _hash
        blocks = [b if _hash.is_string_column(b) else vaex.array_types.to_numpy(b, strict=False) for b in blocks]  # arrow -> numpy like vaex/cpu.py:691
        sel = [None if s is None else vaex.array_types.to_numpy(s) for s in selection_masks]
        return super().process(thread_index, i1, i2, filter_mask, sel, blocks)


class VaexTaskPartHashmapUniqueCreate(_tp.TaskPartHashmapUniqueCreate):
    snake_name = "hash_map_unique_create"

    @classmethod
    def decode(cls, encoding, spec, df, nthreads):
        dtype = _np_dtype(encoding, spec["dtype"])
        dtype_item = _np_dtype(encoding, spec["dtype_item"])
        if dtype_item.kind in "SU" or getattr(encoding.decode("dtype", spec["dtype_item"]), "is_string", False):
            dtype = dtype_item = np.dtype("O")  # string keys: ordered_set_string on the device (csrc/hashset.cu)
        elif dtype.kind == "O" or dtype_item.kind == "O":
            raise NotImplementedError("groupby on python-object columns is not on the GPU path (there is no CPU fallback)")
        return cls(df, spec["expression"], dtype, dtype_item, flatten=spec["flatten"], limit=spec["limit"], limit_raise=spec["limit_raise"],
                   selection=spec["selection"], return_inverse=spec["return_inverse"], nthreads=nthreads)

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        import vaex.array_types
        from . import hash as _hash
        blocks = [b if _hash.is_string_column(b) else vaex.array_types.to_numpy(b, strict=False) for b in blocks]  # strings stay arrow
        return super().process(thread_index, i1, i2, filter_mask, selection_masks, blocks)


class VaexTaskPartStatistic(_tp.TaskPartStatistic):
    """"legacy_statistic" (vaex/cpu.py:487-626): TaskStatistic — df.cov / df.correlation / binned df.minmax and the limits pre-pass of
    df.count(binby=..., limits=None) (vaex/dataframe.py:1519-1521)."""
    snake_name = "legacy_statistic"

    def process(self, thread_index, i1, i2, filter_mask, selection_masks, blocks):
        import vaex.array_types
        blocks = [vaex.array_types.to_numpy(b, strict=False) for b in blocks]
        sel = [None if s is None else vaex.array_types.to_numpy(s) for s in selection_masks]
        return super().process(thread_index, i1, i2, filter_mask, sel, blocks)


_ORIGINAL = {}


def install(legacy_statistic=False):
    """Swap the two task parts in vaex's registry — and with ``legacy_statistic=True`` also "legacy_statistic" (TaskStatistic);
    returns the replaced classes so `uninstall` can restore them."""
    import vaex.cpu
    _ORIGINAL["aggregations"] = vaex.cpu.TaskPartAggregation
    _ORIGINAL["hash_map_unique_create"] = vaex.cpu.TaskPartHashmapUniqueCreate
    vaex.cpu.register(VaexTaskPartAggregation)
    vaex.cpu.register(VaexTaskPartHashmapUniqueCreate)
    if legacy_statistic:
        _ORIGINAL["legacy_statistic"] = vaex.cpu.TaskPartStatistic
        vaex.cpu.register(VaexTaskPartStatistic)
    return dict(_ORIGINAL)


def uninstall():
    import vaex.cpu
    for cls in _ORIGINAL.values():
        vaex.cpu.register(cls)
    _ORIGINAL.clear()
