"""A numpy restatement of the argsort of df.sort (csrc/sort.cu): every key becomes a class digit (value 0, NaN 1, null 2, never
inverted) and an order-preserving unsigned word (zero outside class 0), and np.lexsort over those gives the permutation.
test_sort_oracle_cpu.py pins it to pa.compute.sort_indices, the reference's argsort (vaex/dataframe.py:4694-4745), so the device
test can compare its permutation with arrow's exactly.

A key is (values, mask or None, descending).  Values are numpy arrays of any of the 11 numeric dtypes, datetime64 / timedelta64
(either byte order), or strings (an object array, None = null).  to_arrow converts them the way vaex's to_arrow_table does."""
import numpy as np


def to_arrow(values, mask=None):
    """vaex.array_types.to_arrow (vaex/array_types.py:176-184): native byte order, then pa.array; a mask makes nulls (and then only
    the mask decides: an unmasked NaT stays the value INT64_MIN)"""
    import pyarrow as pa
    values = np.asarray(values)
    if values.dtype.kind == "O":
        return pa.array([None if (mask is not None and m) else v for v, m in zip(values, mask if mask is not None else [False] * len(values))],
                        type=pa.string())
    values = values.astype(values.dtype.newbyteorder("="))
    return pa.array(np.ma.array(values, mask=mask) if mask is not None else values)


def encode(values, mask=None, descending=False):
    """(value word uint64, class uint8) of one key"""
    values = np.asarray(values)
    n = len(values)
    cls = np.zeros(n, np.uint8)
    if values.dtype.kind == "O":
        null = np.array([v is None for v in values], bool)
        if mask is not None:
            null |= np.asarray(mask, bool)
        raw = [v.encode("utf8") if isinstance(v, str) else b"" for v in values]
        distinct = sorted(set(r for r, z in zip(raw, null) if not z))
        rank = {r: i for i, r in enumerate(distinct)}
        w = np.array([rank.get(r, 0) if not z else 0 for r, z in zip(raw, null)], np.uint64)
        full = np.uint64(2 ** 63 - 1)
        cls[null] = 2
    else:
        a = values.astype(values.dtype.newbyteorder("="))
        bits = 8 * a.dtype.itemsize
        full = np.uint64(2 ** bits - 1)
        top = np.uint64(1 << (bits - 1))
        if a.dtype.kind == "f":
            cls[np.isnan(a)] = 1
            a = np.where(a == 0, np.zeros(1, a.dtype), a)  # -0.0 == +0.0
            u = a.view(f"u{a.dtype.itemsize}").astype(np.uint64)
            w = np.where(u & top, ~u & full, u | top)
        elif a.dtype.kind in "iMm":
            a = a.view(f"i{a.dtype.itemsize}")
            if values.dtype.kind in "Mm" and mask is None:
                cls[a == np.iinfo(np.int64).min] = 2  # NaT without a mask is arrow's null
            w = a.view(f"u{a.dtype.itemsize}").astype(np.uint64) ^ top
        elif a.dtype.kind == "b":
            w, full = a.astype(np.uint64), np.uint64(1)
        else:
            w = a.astype(np.uint64)
    if mask is not None:
        cls[np.asarray(mask, bool)] = 2
    if descending:
        w = ~w & full
    w = np.where(cls > 0, np.uint64(0), w).astype(np.uint64)
    return w, cls


def argsort(keys):
    """the stable permutation that sorts rows by keys[0], then keys[1], ...: keys = [(values, mask, descending)]"""
    seq = []
    for values, mask, descending in reversed(keys):
        seq += list(encode(values, mask, descending))  # np.lexsort: the last array is the primary key
    return np.lexsort(seq) if seq else np.zeros(0, np.int64)


def arrow_argsort(keys):
    """pa.compute.sort_indices over the keys' arrow table, as the reference runs it"""
    import pyarrow as pa
    import pyarrow.compute as pc
    table = pa.table({f"k{i}": to_arrow(v, m) for i, (v, m, _) in enumerate(keys)})
    sort_keys = [(f"k{i}", "descending" if d else "ascending") for i, (_, _, d) in enumerate(keys)]
    return pc.sort_indices(table, sort_keys=sort_keys).to_numpy().astype(np.int64)


# ---- the edge corpus ---------------------------------------------------------------------------------------------------------------
NUMERIC = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"]
TIMES = ["datetime64[ns]", "timedelta64[s]"]


def edge_values(dtype):
    """the edge values of a dtype: its limits, zero, ±0.0, ±inf, NaN payloads, subnormals, uint64 at and above 2^63, NaT"""
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return np.array([False, True])
    if dt.kind == "f":
        info = np.finfo(dt)
        nan_bits = [0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001] if dt.itemsize == 8 else [0x7FC00001, 0xFFC00000, 0x7F800001]
        nans = np.array(nan_bits, f"u{dt.itemsize}").view(dt)
        vals = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5, info.max, info.min, info.tiny, -info.tiny, info.smallest_subnormal,
                         -info.smallest_subnormal], dt)
        return np.concatenate([vals, nans])
    if dt.kind in "mM":
        return np.array([0, 5, -5, np.iinfo(np.int64).min, np.iinfo(np.int64).max, np.iinfo(np.int64).min + 1], np.int64).view(dt)
    info = np.iinfo(dt)
    vals = [info.min, info.max, 0, 1, info.max - 1]
    if dt.kind == "i":
        vals += [-1, info.min + 1]
    if dt == np.uint64:
        vals += [2 ** 63, 2 ** 63 - 1, 2 ** 63 + 1]
    return np.array(vals, dt)


STRINGS = np.array(["", "B", "a", "b", "ä", "ab", "a\x00", "zz", "日本", None], dtype=object)


def random_key(rng, dtype, n, masked, byteswap, descending):
    """one corpus key: n rows drawn from the dtype's edge values"""
    if dtype == "string":
        values = rng.choice(STRINGS, n)
    else:
        values = rng.choice(edge_values(dtype), n)
        if byteswap and values.dtype.itemsize > 1:
            values = values.astype(values.dtype.newbyteorder("S"))
    mask = rng.random(n) < 0.2 if masked else None
    return values, mask, descending
