"""Vectorised numpy references for the row-mover edge tests (test_gpu_row_movers_edges.py), fast at millions of rows; both are
pinned to the slower restatements they stand for by test_row_movers_oracle_cpu.py.

- string_key / encode: a sort_oracle string key drawn as codes into sort_oracle.STRINGS, so its encoding is a table lookup instead
  of a Python loop over the rows; argsort takes such keys next to sort_oracle's numeric ones.
- agg_list: AggList_<T>_int64 (csrc/list.cu) restated as the device computes it — one record per row, key cell * 4 + category
  (0 value, 1 NaN, 2 null), rows a call does not keep skipped, one stable sort by key in (call, row) order — against
  oracle.agg_list, which appends to per-cell Python lists."""
import numpy as np

import sort_oracle as S

_PRESENT = [s for s in S.STRINGS if s is not None]
# the bytewise rank of every STRINGS entry (a null entry ranks 0: its word is zeroed anyway)
_RANK = np.array([sorted(s.encode("utf8") for s in _PRESENT).index(s.encode("utf8")) if s is not None else 0 for s in S.STRINGS], np.uint64)
_NULL = np.array([s is None for s in S.STRINGS])


def string_key(rng, n, masked, descending):
    """(values (object array of STRINGS), mask or None, descending, codes into STRINGS)"""
    codes = rng.integers(0, len(S.STRINGS), n)
    mask = rng.random(n) < 0.2 if masked else None
    return S.STRINGS[codes], mask, descending, codes


def arrow_strings(key):
    """a string_key as a pyarrow string array: null where the entry is None or masked"""
    import pyarrow as pa
    _, mask, _, codes = key
    null = _NULL[codes] if mask is None else (_NULL[codes] | mask)
    return pa.array(list(S.STRINGS), type=pa.string()).take(pa.array(codes.astype(np.int32), mask=null))


def encode(key):
    """(value word, class) of a key: sort_oracle.encode for a 3-tuple, the table lookup for a string_key"""
    if len(key) == 3:
        return S.encode(*key)
    _, mask, descending, codes = key
    cls = np.where(_NULL[codes], 2, 0).astype(np.uint8)
    if mask is not None:
        cls[mask] = 2
    w = _RANK[codes]
    if descending:
        w = ~w & np.uint64(2 ** 63 - 1)
    return np.where(cls > 0, np.uint64(0), w).astype(np.uint64), cls


def argsort(keys):
    """sort_oracle.argsort over keys that may include string_keys.  A key whose value words stay below 2^62 sorts as one array, its
    class in the top two bits (the word is zero outside class 0), which halves np.lexsort's passes for the narrow dtypes."""
    seq = []
    for key in reversed(keys):
        w, cls = encode(key)
        if len(w) and int(w.max()) < 2 ** 62:
            seq.append(w | (cls.astype(np.uint64) << np.uint64(62)))
        else:
            seq += [w, cls]
    return np.lexsort(seq)


def call_starts(n, calls):
    """the first row of the bin() call every row belongs to"""
    starts = np.zeros(n, np.int64)
    for i1, i2 in calls:
        starts[i1:i2] = i1
    return starts


def agg_list(cells, values, valid, ncells, dropnan, dropnull, calls):
    """AggList_<T>_int64 over the rows fed as bin() calls `calls` (consecutive, covering every row) -> (int64 offsets[ncells + 1],
    values in native byte order, bool per value: a null slot (its value unspecified)).  `valid`: 1 = use the row, 0 = null, None
    = all; row r of a call is judged by valid[r % 1024] of that call, the reference's quirk."""
    cells = np.asarray(cells, np.int64)
    a = np.asarray(values)
    a = a.astype(a.dtype.newbyteorder("="))
    n = len(cells)
    starts = call_starts(n, calls)
    v = np.ones(n, np.uint8) if valid is None else np.asarray(valid)[starts + (np.arange(n) - starts) % 1024]
    nan = np.isnan(a) if a.dtype.kind == "f" else np.zeros(n, bool)
    cat = np.full(n, -1, np.int64)
    cat[(v == 1) & ~nan] = 0
    if not dropnan:
        cat[(v == 1) & nan] = 1
    if not dropnull:
        cat[v == 0] = 2
    kept = np.flatnonzero(cat >= 0)
    order = kept[np.argsort(cells[kept] * 4 + cat[kept], kind="stable")]
    offsets = np.zeros(ncells + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(cells[kept], minlength=ncells))
    out = a[order].copy()
    if a.dtype.kind == "f":
        out[cat[order] == 1] = np.nan  # the canonical quiet NaN, whatever the row's payload
    out[cat[order] == 2] = 0
    return offsets, out, cat[order] == 2
