"""The chunk-feed loop — GPU restatement of ExecutorLocal for this path.

Reference: packages/vaex-core/vaex/execution.py:141-169 (_merge_tasks_for_df: aggregations with EQUAL binner tuples share
one grid and one pass), :283-292 (chunk_size_for), :385-412 (task -> task part, ideal_splits, see_all), :432-435 (thread pool
map over dataset.chunk_iterator), :451-453 (reduce + get_result); vaex/multithreading.py:64-80 (stable thread index).

Two feeds:
  * host columns (numpy): chunks go to a pool of `nthreads` workers; worker t always uses slot t (its own CUDA stream and
    H2D staging arena), so copies of one chunk overlap the kernels of another — the role the GIL-free C++ sections play
    in the reference.
  * device columns (``__cuda_array_interface__``, e.g. torch CUDA tensors): ONE call over the whole row range — the
    roofline configuration; no chunking, no host involvement per row.
"""
import math
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib
from . import taskpart as _tp


class Task:
    """What the executor needs from a task: expressions (column names), optional selections (mask arrays) and a part."""

    def __init__(self, part, selections=()):
        self.part = part
        self.expressions = list(part.expressions)
        self.selections = list(selections)
        self.result = None
        self.stopped = False
        self.cancelled = False


class Executor:
    def __init__(self, nthreads=None, chunk_size=None, chunk_size_min=1024, chunk_size_max=16 * 1024 * 1024):
        # the reference caps chunks at 1M rows (vaex/settings.py:85-87); a GPU wants >= 16M-row chunks to amortise launches,
        # so the cap is larger here.  Pass chunk_size_max=1024**2 to reproduce the reference's chunking exactly.
        self.nthreads = nthreads or min(8, os.cpu_count() or 1)
        self.chunk_size = chunk_size
        self.chunk_size_min = chunk_size_min
        self.chunk_size_max = chunk_size_max
        self.passes = 0

    def chunk_size_for(self, row_count):
        # vaex/execution.py:283-292
        if self.chunk_size is not None:
            return self.chunk_size
        one_pass = math.ceil(row_count / self.nthreads) if row_count else 1
        return min(self.chunk_size_max, max(self.chunk_size_min, one_pass))

    def execute(self, columns, tasks, row_count=None, i0=0, progress=None, filter=None):
        """One pass over `columns` (dict name -> array) feeding every task part; returns [task.result...].

        filter: a device-evaluated boolean expression (expression.DeviceExpression).  Per chunk the mask is computed on the
                worker's slot and EVERY dependent column — and every selection mask — is compacted with it on the device before
                the task parts see a row (vaex/execution.py:516-522); the parts get ``filter_mask`` and blocks of the kept length.
        progress: called with the fraction done after every chunk; a return value of exactly ``False`` cancels the pass
                (vaex/multithreading.py:111-118): no further chunk is fed, the tasks are marked cancelled and UserAbort is raised
                (vaex/execution.py:478-482)."""
        if not tasks:
            return []
        needed = sorted({e for t in tasks for e in t.expressions})
        for e in needed:
            if e not in columns:
                raise KeyError(f"column {e!r} not found")
        if row_count is None:
            row_count = len(columns[needed[0]]) if needed else 0
        self.passes += 1
        # memory pre-declaration cross-check (vaex/execution.py:413-414): what the parts report must be what their aggregators hold
        for t in tasks:
            declared = getattr(t.part, "predicted_memory_usage", None)
            if declared is not None and declared != t.part.memory_usage():
                raise RuntimeError(f"Reported memory usage by tasks was {t.part.memory_usage()}, while tracker listed {declared}")

        feed_cols = [columns[e] for e in needed] + ([filter] if filter is not None else []) + [s for t in tasks for s in t.selections if s is not None]
        device = bool(feed_cols) and all(_lib.on_device(c) for c in feed_cols)
        errors = []
        cancelled = threading.Event()

        def feed(thread_index, i1, i2):
            if cancelled.is_set():
                return 0
            live = [t for t in tasks if not (t.stopped or t.part.stopped)]
            for t in tasks:
                if t.part.stopped:
                    t.stopped = True
            raw = {e: _lib.chunk_of(columns[e], thread_index, i1, i2) for e in sorted({e for t in live for e in t.expressions})}
            sels = {id(s): _lib.chunk_of(s, thread_index, i1, i2) for t in live for s in t.selections if s is not None}
            filter_mask = None
            if filter is not None and live:
                from . import expression as _expr
                filter_mask = filter.chunk(thread_index, i1, i2)
                names, sel_ids = list(raw), list(sels)
                kept, out = _expr.compact(thread_index, filter_mask, [raw[k] for k in names] + [_as_u8(sels[k]) for k in sel_ids])
                raw = dict(zip(names, out[:len(names)]))
                sels = dict(zip(sel_ids, out[len(names):]))
                filter_mask.kept = kept  # count(*) has no block to take its length from
            for t in live:
                blocks = [raw[e] for e in t.expressions]
                sel = [None if s is None else sels[id(s)] for s in t.selections]
                try:
                    if filter_mask is None or filter_mask.kept:
                        t.part.process(thread_index, i0 + i1, i0 + i2, filter_mask, sel, blocks)
                except Exception as e:  # stash and re-raise on the main thread (vaex/execution.py:567-571)
                    errors.append(e)
                    t.stopped = True
            if progress is not None and progress(i2 / max(row_count, 1)) is False:
                cancelled.set()
            return i2 - i1

        if row_count:
            if device:
                feed(0, 0, row_count)
            else:
                chunk = self.chunk_size_for(row_count)
                ranges = [(i, min(i + chunk, row_count)) for i in range(0, row_count, chunk)]
                if self.nthreads == 1 or len(ranges) == 1:
                    for r in ranges:
                        feed(0, *r)
                else:
                    local = threading.local()
                    lock = threading.Lock()
                    counter = [0]

                    def work(r):  # ThreadPoolIndex: every worker keeps one index for its lifetime
                        if not hasattr(local, "index"):
                            with lock:
                                local.index = counter[0]
                                counter[0] += 1
                        return feed(local.index, *r)

                    with ThreadPoolExecutor(self.nthreads) as pool:
                        list(pool.map(work, ranges))
        if errors:
            raise errors[0]
        if cancelled.is_set():
            for t in tasks:
                t.cancelled = True
            raise UserAbort("Task was cancelled")
        for t in tasks:
            t.part.reduce([])
            t.result = t.part.get_result()
        return [t.result for t in tasks]


def _as_u8(mask):
    """selection masks travel as one byte per row"""
    mask = _lib.unmask_selection(mask)
    if _lib.is_device(mask):
        return mask
    return np.ascontiguousarray(mask).astype(np.bool_, copy=False).view(np.uint8)


class UserAbort(Exception):
    """vaex.execution.UserAbort: raised when a progress callback returned False"""


def merge_aggregation_tasks(requests, dtypes, nthreads):
    """_merge_tasks_for_df (vaex/execution.py:141-169): requests = [(binner_specs, descriptor, selection_masks)];
    every group with an equal binner tuple becomes ONE TaskPartAggregation (one pass, one set of binners)."""
    groups = {}
    order = []
    for binner_specs, desc, sel in requests:
        key = tuple(tuple(sorted((k, str(v)) for k, v in b.items() if k != "hash_map_unique") + [("hm", id(b.get("hash_map_unique")))]) for b in binner_specs)
        if key not in groups:
            groups[key] = (binner_specs, [], [])
            order.append(key)
        groups[key][1].append(desc)
        groups[key][2].append(sel)
    tasks = []
    index = []  # request -> (task, position)
    for key in order:
        binner_specs, descs, sels = groups[key]
        for d in descs:
            d._prepare_types(dtypes)
        binners = [_tp.decode_binner(b, nthreads) for b in binner_specs]
        part = _tp.TaskPartAggregation(None, binners, descs, dtypes, nthreads=nthreads)
        selections = []
        for d, s in zip(descs, sels):
            d_sel = d.selection if isinstance(d.selection, (list, tuple)) else [d.selection]
            for i, one in enumerate(d_sel):
                selections.append(None if one is None or one is False else (s[i] if isinstance(s, (list, tuple)) else s))
        tasks.append(Task(part, selections))
    pos = {}
    for binner_specs, desc, sel in requests:
        pos[id(desc)] = None
    for t in tasks:
        for k, d in enumerate(t.part.aggregation_descriptions):
            pos[id(d)] = (t, k)
    return tasks, pos
