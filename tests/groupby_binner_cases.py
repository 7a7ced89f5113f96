"""vaex's own tests of the groupby binners (tests/groupby_test.py:276-300, 380-423, 608-636 and tests/agg_test.py:611-712 of the reference)
restated as data.  A case is (name, columns, keys, agg, expected, kwargs): `keys` lists ("time", column, resolution, every),
("binner", column, vmin, vmax, bins), ("integer", column, {BinnerInteger keywords}) or a column name; `agg` is ("count",), ("sum", col),
("nunique", col) or ("list", col); `expected` maps an output column to the reference's values (None = the null group) or, for a list,
to the set of the first group's elements.  `numpy_groupby` computes the same outputs with numpy alone."""
import numpy as np

LARGE = 2 ** 16
OFFSET = 2 ** 16


def _days(a, b):
    return np.arange(a, b, dtype="M8[D]")


def _ma(values, dtype):
    return np.ma.array([0 if v is None else v for v in values], mask=[v is None for v in values], dtype=dtype)


_T1, _T2 = _days("2015-01-01", "2015-02-01"), _days("2015-01-01", "2016-01-02")
_Y1 = np.arange(len(_T1))

CASES = [
    ("datetime_per_week", {"t": _T1, "y": _Y1}, [("time", "t", "W", 1)], ("sum", "y"),
     {"y": [int(_Y1[k * 7:(k + 1) * 7].sum()) for k in range(5)]}, {}),
    ("datetime_quarter", {"t": _T2, "y": np.arange(len(_T2))}, [("time", "t", "M", 3)], ("sum", "y"),
     {"__len__": 5, "__sum__": int(np.arange(len(_T2)).sum())}, {}),
    ("int8_dropmissing", {"g": _ma([-10, 1, 1, 127, None], "int8"), "x": np.array([3, 2, 2, 5, 6])}, [("integer", "g", {"dropmissing": True})],
     ("sum", "x"), {"g": [-10, 1, 127], "sum": [3, 4, 5]}, {}),
    ("int8_with_null", {"g": _ma([-10, 1, 1, 127, None], "int8"), "x": np.array([3, 2, 2, 5, 6])}, [("integer", "g", {})],
     ("sum", "x"), {"g": [-10, 1, 127, None], "sum": [3, 4, 5, 6]}, {}),
    ("int_binner_with_null_ascending", {"g": _ma([-10, 1, 1, 127, LARGE, None], "int64"), "x": _ma([3, None, 4, 5, 99, 6], "int64")},
     [("integer", "g", {"min_value": -10, "max_value": LARGE, "sort": True, "ascending": True})], ("sum", "x"),
     {"g": [-10, 1, 127, LARGE, None], "sum": [3, 4, 5, 99, 6]}, {}),
    ("int_binner_with_null_descending", {"g": _ma([-10, 1, 1, 127, LARGE, None], "int64"), "x": _ma([3, None, 4, 5, 99, 6], "int64")},
     [("integer", "g", {"min_value": -10, "max_value": LARGE, "sort": True, "ascending": False})], ("sum", "x"),
     {"g": [LARGE, 127, 1, -10, None], "sum": [99, 5, 4, 3, 6]}, {}),
    ("int_binner_with_offset_2d", {"x": np.array([0, 1, 1, 2], dtype="int32") + OFFSET, "y": np.array([0, 0, 0, 1], dtype="int32")},
     [("integer", "x", {"min_value": OFFSET, "max_value": OFFSET + 2, "sort": True}), ("integer", "y", {"min_value": 0, "max_value": 1, "sort": True})],
     ("sum", "x"), {"x": [OFFSET, OFFSET + 1, OFFSET + 2], "y": [0, 0, 1], "sum": [OFFSET, (OFFSET + 1) * 2, OFFSET + 2]}, {}),
    ("binner_1d", {"x": np.array([0.1, 1.1, 1.2, 2.2, 2.5, 2.7])}, [("binner", "x", 0, 3, 3)], ("count",),
     {"x": [0.5, 1.5, 2.5], "count": [1, 2, 3]}, {}),
    ("binner_2d", {"x": np.array([0.1, 1.1, 1.2, 2.2, 2.5, 2.7, 100]), "g": np.array([0, 0, 1, 0, 1, 1, 1])}, [("binner", "x", 0, 3, 3), "g"],
     ("count",), {"x": [0.5, 1.5, 1.5, 2.5, 2.5], "g": [0, 0, 1, 0, 1], "count": [1, 1, 1, 1, 2]}, {"sort": True}),
    ("unique_2d", {"x": np.array([0, 0, 1, 1, 1, 2, 2, 2, 2], dtype="int8"), "y": np.array([4, 5, 4, 5, 5, 4, 5, 5, 5], dtype="int8"),
                   "z": np.array([0, 0, 0, 0, 1, 0, 1, 2, 3])},
     [("integer", "x", {"sort": True}), ("integer", "y", {"sort": True})], ("nunique", "z"),
     {"x": [0, 0, 1, 1, 2, 2], "y": [4, 5, 4, 5, 4, 5], "c": [1, 1, 1, 2, 1, 3]}, {}),
    ("agg_arrow_integer_list", {"x": np.array([0, 0, 0, 0, 0, 1, 1, 1, 2]),
                                "s": np.array(["aap", "aap", "noot", "mies", None, "mies", "kees", "mies", "aap"], dtype=object)},
     [("integer", "x", {"sort": True, "min_value": 0, "max_value": 2})], ("list", "s"),
     {"x": [0, 1, 2], "__first_list__": {"mies", "aap", "noot", None}}, {}),
]


def _key_cells(columns, key):
    """numpy's cells of one key: (group index per row or -1 to drop, group keys)"""
    if isinstance(key, str):
        values = np.asarray(columns[key])
        uniq = np.unique(values)
        return np.searchsorted(uniq, values), list(uniq)
    kind, name = key[0], key[1]
    col = columns[name]
    if kind == "time":
        _, _, res, every = key
        p = col.astype(f"M8[{res}]")
        begin, end = p.min(), p.max()
        idx = (p - begin).astype(np.int64) // every
        return idx, list(np.arange(begin, end + 1, every))
    if kind == "binner":
        _, _, vmin, vmax, bins = key
        x = np.asarray(col, dtype=float)
        idx = np.floor((x - vmin) / (vmax - vmin) * bins).astype(np.int64)
        idx[(x < vmin) | (x >= vmax)] = -1
        return idx, list(vmin + (np.arange(bins) + 0.5) * (vmax - vmin) / bins)
    kw = key[2]
    values, mask = np.ma.getdata(col).astype(np.int64), np.ma.getmaskarray(col)
    lo = kw.get("min_value", -128 if col.dtype == np.int8 else 0)
    hi = kw.get("max_value", 127 if col.dtype == np.int8 else 255)
    n = hi - lo + 1
    idx = values - lo
    null = mask | (idx < 0) | (idx >= n)
    desc = kw.get("sort") and not kw.get("ascending", True)
    idx = np.where(null, n, (n - 1 - idx) if desc else idx)
    keys = (list(range(hi, lo - 1, -1)) if desc else list(range(lo, hi + 1))) + [None]
    if kw.get("dropmissing"):
        idx[null] = -1
        keys = keys[:-1]
    return idx, keys


def numpy_groupby(columns, keys, agg):
    """the groups with rows, in key order (first key slowest), and the aggregate of each"""
    cells = [_key_cells(columns, k) for k in keys]
    n = len(next(iter(columns.values())))
    rows = {}
    for r in range(n):
        cell = tuple(int(c[0][r]) for c in cells)
        if min(cell) >= 0:
            rows.setdefault(cell, []).append(r)
    out = {"keys": [], "values": []}
    for cell in sorted(rows):
        out["keys"].append(tuple(c[1][i] for c, i in zip(cells, cell)))
        rs = rows[cell]
        if agg[0] == "count":
            out["values"].append(len(rs))
            continue
        col = columns[agg[1]]
        vals = [None if np.ma.getmaskarray(col)[r] else col[r] for r in rs] if np.ma.isMaskedArray(col) else [col[r] for r in rs]
        if agg[0] == "sum":
            out["values"].append(int(sum(v for v in vals if v is not None)))
        elif agg[0] == "nunique":
            out["values"].append(len(set(vals)))
        else:
            out["values"].append(list(vals))
    return out
