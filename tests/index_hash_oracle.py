"""Restatement of index_hash<T> (reference src/hash_primitives.hpp:731-1040) under the sequential rule the device follows.

* primary row of a key = its smallest row ``start_index + i`` over all updates and merges;
* overflow = the key's other rows, ascending;
* NaN / null row = the largest NaN / null row seen (global, ``start_index`` included);
* has_duplicates = some non-NaN, non-null key occurs more than once;
* merge = the union of both indexes' rows under the same rules.

For one ``update`` at ``start_index=0``, and for several calls with increasing ``start_index`` and no NaN / null, this is what the
reference computes.  Elsewhere the reference differs (DESIGN.md, index_hash): its NaN / null row is call-local, a merge drops the
other index's NaN / null row, does not set has_duplicates by itself and appends the overflow in merge order.

``IndexHash(dtype, nmaps, bits=True)`` keys floats by their canonical bit pattern (set_cases.canon), as the device does: -0.0 and 0.0
are two keys there.  Lookups are first cast by value to the index's dtype, as the host's map_index does.  The default keys by Python
``==`` (so -0.0 == 0.0), which is what the reference's std::equal_to does.
"""
import numpy as np

from set_cases import canon


class IndexHash:
    def __init__(self, dtype, nmaps=1, bits=False):
        self.dtype = np.dtype(dtype)
        self.nmaps = nmaps
        self.bits = bits
        self.rows = {}  # key -> every row, unsorted
        self.nan_count = self.null_count = 0
        self.nan_row = self.null_row = None

    def _keys(self, values):
        a = np.asarray(values)
        if a.dtype != self.dtype:
            with np.errstate(invalid="ignore", over="ignore"):
                a = a.astype(self.dtype)  # update force-casts (py::array_t<T> forcecast)
        return a

    def _hashable(self, a):
        """the dict keys of a key array: its values, or in bit-pattern mode the canonical patterns of its values in the index's dtype"""
        if not self.bits:
            return a.tolist()
        if a.dtype != self.dtype:
            with np.errstate(invalid="ignore", over="ignore"):
                a = a.astype(self.dtype)
        return canon(a).tolist()

    def update(self, values, mask=None, start_index=0):
        a = self._keys(values)
        isnan = np.isnan(a) if a.dtype.kind == "f" else np.zeros(len(a), bool)
        m = np.zeros(len(a), bool) if mask is None else np.asarray(mask).astype(bool)
        for i, (k, nan, masked) in enumerate(zip(self._hashable(a), isnan.tolist(), m.tolist())):
            row = start_index + i
            if masked:
                self.null_count += 1
                self.null_row = row if self.null_row is None else max(self.null_row, row)
            elif nan:
                self.nan_count += 1
                self.nan_row = row if self.nan_row is None else max(self.nan_row, row)
            else:
                self.rows.setdefault(k, []).append(row)

    def merge(self, other):
        for k, r in other.rows.items():
            self.rows.setdefault(k, []).extend(r)
        self.nan_count += other.nan_count
        self.null_count += other.null_count
        for name in ("nan_row", "null_row"):
            mine, theirs = getattr(self, name), getattr(other, name)
            if theirs is not None:
                setattr(self, name, theirs if mine is None else max(mine, theirs))

    def _specials(self):
        return int(self.nan_count > 0) + int(self.null_count > 0)

    def __len__(self):
        return sum(len(r) for r in self.rows.values()) + self._specials()

    @property
    def count(self):
        return len(self.rows) + self._specials()

    @property
    def has_duplicates(self):
        return any(len(r) > 1 for r in self.rows.values())

    def map_index(self, values, mask=None):
        """(int64 rows, encountered_unknown)"""
        a = np.asarray(values)
        isnan = np.isnan(a) if a.dtype.kind == "f" else np.zeros(len(a), bool)
        m = np.zeros(len(a), bool) if mask is None else np.asarray(mask).astype(bool)
        out = np.full(len(a), -1, np.int64)
        unknown = False
        for i, (k, nan, masked) in enumerate(zip(self._hashable(a), isnan.tolist(), m.tolist())):
            if nan:
                v = self.nan_row if self.nan_count else -1
            elif masked:
                v = self.null_row if self.null_count else -1
            else:
                r = self.rows.get(k)
                v = min(r) if r else -1
                unknown |= not r
                out[i] = v
                continue
            unknown |= v == -1
            out[i] = v
        return out, unknown

    def map_index_duplicates(self, values, start_index, mask=None):
        a = np.asarray(values)
        isnan = np.isnan(a) if a.dtype.kind == "f" else np.zeros(len(a), bool)
        m = np.zeros(len(a), bool) if mask is None else np.asarray(mask).astype(bool)
        left, right = [], []
        for i, (k, nan, masked) in enumerate(zip(self._hashable(a), isnan.tolist(), m.tolist())):
            if nan or masked or k not in self.rows:
                continue
            extra = sorted(self.rows[k])[1:]
            left += [start_index + i] * len(extra)
            right += extra
        return np.array(left, np.int64), np.array(right, np.int64)

    def extract(self):
        """{key: primary row} over all shards (the shard split is the reference's hash; compare the union); in bit-pattern mode the
        keys are canonical patterns"""
        return {k: min(r) for k, r in self.rows.items()}


def truncate(rows, out_dtype):
    """the reference's assignment of an int64 row into an int8..int64 `out` array"""
    return np.asarray(rows, np.int64).astype(out_dtype)


class RefAPI(IndexHash):
    """the restatement behind the reference's method signatures (update overloads, map_index with `out`), so one driver can run the
    compiled reference, the device classes and this"""

    def update(self, values, *args):
        args = list(args)
        mask = args.pop(0) if args and isinstance(args[0], np.ndarray) else None
        IndexHash.update(self, values, mask, args[0] if args else 0)

    def _write(self, rows, unknown, out):
        if out is None:
            return rows
        out[:] = truncate(rows, out.dtype)
        return unknown

    def map_index(self, values, out=None):
        return self._write(*IndexHash.map_index(self, values), out)

    def map_index_masked(self, values, mask, out=None):
        return self._write(*IndexHash.map_index(self, values, mask), out)


def classes(dtype, bits=False):
    return lambda nmaps=1: RefAPI(dtype, nmaps, bits)
