"""Restatement of DataFrameLocal.join (reference vaex/join.py:125-297) in numpy, over the index restatement of index_hash_oracle.

A frame here is ``OFrame(columns, filter)``: columns are numpy / numpy.ma arrays (object arrays for strings, None = missing) and the
filter is a boolean array over the rows, or None.  Virtual columns and expression keys are passed as evaluated columns.  The index
follows the sequential rule (index_hash_oracle), and where the reference's answer depends on thread timing or differs for another
reason this restatement gives the answer the device gives (DESIGN.md section 3, join):

1. the appended duplicate rows are ordered by (left row, right overflow row);
2. has_duplicates follows the sequential rule;
3. a masked left key maps to the right's null row and adds no duplicate pairs;
4. with a filtered left and duplicates, the unfiltered rows are taken.
"""
import numpy as np

from index_hash_oracle import IndexHash


class OFrame:
    def __init__(self, columns, filter=None, variables=None):
        self.columns = dict(columns)
        self.filter = None if filter is None else np.asarray(filter, bool)
        self.variables = dict(variables or {})
        lengths = {len(c) for c in self.columns.values()}
        assert len(lengths) <= 1
        self.length = lengths.pop() if lengths else 0

    def __len__(self):
        return self.length

    def values(self, name, filtered=True):
        """the column as a python list (None = missing), the filter applied"""
        v = self.columns[name]
        v = v if not filtered or self.filter is None else v[self.filter]
        return np.ma.asarray(v).tolist() if np.ma.isMaskedArray(v) else np.asarray(v).tolist()


def take(col, rows):
    """col[rows] with rows < 0 missing: a masked array when a row is missing or the column was masked"""
    rows = np.asarray(rows, np.int64)
    missing = rows < 0
    safe = np.where(missing, 0, rows)
    data = np.ma.getdata(col)[safe] if len(col) else np.zeros(len(rows), np.ma.getdata(col).dtype)
    mask = missing | (np.ma.getmaskarray(col)[safe] if len(col) else missing)
    if data.dtype.kind == "O":
        data = data.copy()
        data[mask] = None
    elif missing.any():
        data = data.copy()
        data[missing] = 0
    if np.ma.isMaskedArray(col) or mask.any():
        return np.ma.array(data, mask=mask)
    return data


def concat(a, b):
    if np.ma.isMaskedArray(a) or np.ma.isMaskedArray(b):
        return np.ma.concatenate([np.ma.asarray(a), np.ma.asarray(b)])
    return np.concatenate([a, b])


def extract(f):
    if f.filter is None:
        return OFrame(f.columns, variables=f.variables)
    return OFrame({k: v[f.filter] for k, v in f.columns.items()}, variables=f.variables)


def _keys(col):
    data, mask = np.ma.getdata(col), (np.ma.getmaskarray(col) if np.ma.isMaskedArray(col) else None)
    if data.dtype.kind in "mM":
        data = data.view(np.int64)
    return data, mask


def required_dtype_for_max(n):
    for dtype in (np.int8, np.int16, np.int32, np.int64):
        if n <= np.iinfo(dtype).max:
            return np.dtype(dtype)


def find_valid_name(name, used):
    if name in used:
        nr = 1
        while name + ("_%d" % nr) in used:
            nr += 1
        name = name + ("_%d" % nr)
    return name


def mangle_name(prefix, name, suffix):
    if name.startswith("__"):
        return "__" + prefix + name[2:] + suffix
    return prefix + name + suffix


def join(df, other, on=None, left_on=None, right_on=None, lprefix='', rprefix='', lsuffix='', rsuffix='', how='left', allow_duplication=False,
         bits=False):
    """`bits`: key the index by bit pattern, the device's rule (index_hash_oracle.IndexHash)"""
    inner = False
    left, right = df, other
    if how == 'left':
        pass
    elif how == 'right':
        left, right = right, left
        lprefix, rprefix = rprefix, lprefix
        lsuffix, rsuffix = rsuffix, lsuffix
        left_on, right_on = right_on, left_on
    elif how == 'inner':
        inner = True
    else:
        raise ValueError('join type not supported: {}, only left and right'.format(how))
    left_on = left_on or on
    right_on = right_on or on
    for name in right.columns:
        if left_on and (rprefix + name + rsuffix == lprefix + left_on + lsuffix):
            continue
        if name in left.columns and rprefix + name + rsuffix == lprefix + name + lsuffix:
            raise ValueError('column name collision: {} exists in both column, and no proper suffix given'.format(name))
    right = extract(right)
    lcols = dict(left.columns)
    lfilter = left.filter
    N = left.length
    lookup = None
    if left_on is not None or right_on is not None:
        keys, mask = _keys(right.columns[right_on])
        index = IndexHash(keys.dtype, bits=bits)
        index.update(keys, mask)
        if index.has_duplicates and not allow_duplication:
            raise ValueError('This join will lead to duplication of rows which is disabled, pass allow_duplication=True')
        lkeys, lmask = _keys(left.columns[left_on])
        lookup, _ = index.map_index(lkeys, lmask)
        lookup = lookup.astype(required_dtype_for_max(len(right))).astype(np.int64)
        if index.has_duplicates:
            lookup_left, lookup_right = index.map_index_duplicates(lkeys, 0, lmask)
            if len(lookup_left):
                lcols = {k: concat(v, take(v, lookup_left)) for k, v in lcols.items()}
                if lfilter is not None:
                    lfilter = np.concatenate([lfilter, lfilter[lookup_left]])
                lookup = np.concatenate([lookup, lookup_right])
        if inner:
            matched = np.flatnonzero(lookup != -1)
            lookup = lookup[matched]
            lcols = {k: take(v, matched) for k, v in lcols.items()}
            if lfilter is not None:
                lfilter = lfilter[matched]
    right_names = list(right.columns)
    left_names = list(lcols)
    rcols = dict(right.columns)
    for name in list(right_names):
        if name in left_names:
            all_names = list(set(right_names + left_names))
            all_names.append(mangle_name(lprefix, name, lsuffix))
            all_names.remove(name)
            new_name = mangle_name(rprefix, name, rsuffix)
            if new_name != left_on:
                if new_name in all_names:
                    new_name = find_valid_name(new_name, all_names)
                rcols = {(new_name if k == name else k): v for k, v in rcols.items()}
                right_names[right_names.index(name)] = new_name
            all_names = list(set(right_names + left_names))
            all_names.remove(name)
            new_name = mangle_name(lprefix, name, lsuffix)
            if new_name in all_names:
                new_name = find_valid_name(new_name, all_names)
            lcols = {(new_name if k == name else k): v for k, v in lcols.items()}
            left_names[left_names.index(name)] = new_name
    out = dict(lcols)
    for name, col in rcols.items():
        if name == left_on and name in left_names:
            continue
        assert name not in left_names
        if lookup is None:
            if len(col) != N:
                raise ValueError("a join without a key needs equal row counts")
            out[name] = col
        else:
            out[name] = take(col, lookup)
    variables = dict(left.variables)
    variables.update(right.variables)
    return OFrame(out, lfilter, variables)


def numpy_join(left_keys, right_keys):
    """an argsort-based left join with duplicates: (left rows, right rows) with -1 for no match, ordered like the device join (every
    left row with its primary right row first, then the repeated rows by (left row, right row))"""
    order = np.argsort(right_keys, kind="stable")
    sk = right_keys[order]
    lo = np.searchsorted(sk, left_keys, "left")
    hi = np.searchsorted(sk, left_keys, "right")
    count = hi - lo
    primary = np.where(count > 0, order[np.minimum(lo, len(sk) - 1)], -1)
    extra = np.maximum(count - 1, 0)
    left_rows = np.repeat(np.arange(len(left_keys)), extra)
    starts = np.repeat(lo + 1, extra)
    within = np.arange(extra.sum()) - np.repeat(np.cumsum(extra) - extra, extra)
    right_rows = order[starts + within]
    return np.concatenate([np.arange(len(left_keys)), left_rows]), np.concatenate([primary, right_rows])
