"""Frame.join (vaex/join.py:125-297) and Frame._index (vaex/dataframe.py:514-572) over the device index_hash_<T>.

The right side's key is indexed on the device (taskpart.TaskPartIndex), the left side's key is looked up on the device
(taskpart.TaskPartLookup), and every row move of the join — the right's columns to the left's rows (:286), the left's rows repeated
for the right's duplicates (:214) and the inner join's matched rows (:218-222) — is one b200_take / b200_take_strings gather.

Where the output lands: next to the left key.  A device key gives torch tensors on the device, a host key numpy arrays; string
columns come back as arrow arrays.  A column with a missing row is a host ``np.ma`` array, as Frame has no device-side mask.
"""
import ctypes as C

import numpy as np

from . import _lib, execution, taskpart
from . import hash as _hash

MAX_TAKE_COLUMNS = 16  # b200_take's columns per launch


def _is_virtual(x):
    return getattr(x, "device_virtual", False)


def _torch():
    import torch
    return torch


def _torch_dtype(dtype):
    return _torch().from_numpy(np.empty(0, np.dtype(dtype))).dtype


def _device_tensor(x):
    """a device column as a torch tensor (DeviceArray views included)"""
    torch = _torch()
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(x, device=f"cuda:{_lib.context().device}")


def required_dtype_for_max(n):
    """vaex.utils.required_dtype_for_max (signed): the narrowest integer type holding row numbers up to n"""
    for dtype in (np.int8, np.int16, np.int32, np.int64):
        if n <= np.iinfo(dtype).max:
            return np.dtype(dtype)
    raise ValueError(f"Cannot store a max value of {n} inside an uint64/int64")


def find_valid_name(name, used):
    """vaex.utils.find_valid_name for names already valid: the first `name_<k>` not in `used`"""
    if name in used:
        nr = 1
        while name + ("_%d" % nr) in used:
            nr += 1
        name = name + ("_%d" % nr)
    return name


def mangle_name(prefix, name, suffix):
    """join.py:225-229: a hidden name keeps its leading __"""
    if name.startswith("__"):
        return "__" + prefix + name[2:] + suffix
    return prefix + name + suffix


# ---- the gathers ----------------------------------------------------------------------------------------------------------------
def _staged(x):
    """a column on the device for a gather, as a torch tensor: device columns in place, host ones copied once (bit patterns: datetimes
    and unsigned integers travel as signed integers of their width)"""
    torch = _torch()
    if _lib.is_device(x):
        # torch has no datetime64 / timedelta64: a device datetime column travels as its int64 ticks, as a host one does
        return _device_tensor(_lib.int64_view(x) if _lib.dtype_of(x).kind in "mM" else x)
    a = np.ascontiguousarray(x)
    if a.dtype.kind in "mMu" and a.dtype.itemsize > 1:
        a = a.view(f"i{a.dtype.itemsize}")
    return torch.from_numpy(a).to(f"cuda:{_lib.context().device}")


def _staged_index(index):
    t = _staged(index)
    if t.dtype not in (_torch().int8, _torch().int16, _torch().int32, _torch().int64):
        raise TypeError(f"take: the index must be int8, int16, int32 or int64, not {t.dtype}")
    return t


def _raw_dtype(dtype):
    """the torch dtype a gather writes a column of `dtype` to: its own where torch has it, else a signed integer of its width"""
    dtype = np.dtype(dtype)
    if dtype.kind in "mMu" and dtype.itemsize > 1:
        return _torch_dtype(f"i{dtype.itemsize}")
    return _torch_dtype(dtype)


def take(index, columns, src_len, device):
    """b200_take: [(data, mask or None)] of `src_len` rows each, gathered by `index` (host or device, int8..int64; < 0 = missing).
    Returns [(values, valid or None)]: `valid` (1 = valid, next to the values) only for a column with a missing row.  The values stay
    on the device (torch) when `device` is true and the dtype has a torch equivalent, else they come back as host numpy."""
    torch = _torch()
    ctx = _lib.context()
    ctx.sync()  # device columns may come from a device expression written on a slot's stream
    idx = _staged_index(index)
    n = len(idx)
    results = []
    for k in range(0, len(columns), MAX_TAKE_COLUMNS):
        group = columns[k:k + MAX_TAKE_COLUMNS]
        srcs, masks, outs, valids, dtypes = [], [], [], [], []
        for data, mask in group:
            dt = _lib.dtype_of(data)
            if not dt.isnative:
                data, dt = np.asarray(data).astype(dt.newbyteorder("=")), dt.newbyteorder("=")
            if len(data) != src_len:
                raise ValueError(f"take: a column has {len(data)} rows, expected {src_len}")
            srcs.append(_staged(data))
            masks.append(None if mask is None else _staged(np.asarray(mask).astype(np.uint8)))
            on_device = device and dt.kind not in "mM"
            outs.append(torch.empty(n, dtype=_torch_dtype(dt) if on_device else _raw_dtype(dt), device=idx.device))
            valids.append(torch.empty(n, dtype=torch.uint8, device=idx.device))
            dtypes.append((dt, on_device))
        m = len(group)
        P = C.c_void_p * m
        missing = (C.c_int32 * m)()
        torch.cuda.synchronize(idx.device)  # staging copies and torch-made inputs run on torch's stream, the gather on a slot's
        _lib.check(_lib.lib().b200_take(ctx._h, 0, idx.data_ptr(), idx.element_size(), n, m, P(*[t.data_ptr() for t in srcs]),
                                        (C.c_int32 * m)(*[t.element_size() for t in srcs]), P(*[None if t is None else t.data_ptr() for t in masks]),
                                        int(src_len), P(*[t.data_ptr() for t in outs]), P(*[t.data_ptr() for t in valids]), missing))
        for i, (out, valid, (dt, on_device)) in enumerate(zip(outs, valids, dtypes)):
            if not on_device:
                out = out.cpu().numpy().view(dt)
                valid = valid.cpu().numpy()
            results.append((out, valid if missing[i] else None))
    return results


def _string_source(values):
    """an arrow string / large_string array (or numpy object strings) -> (offsets, offset itemsize, bytes, first, mask or None).  `bytes`
    are the rows' own bytes: offsets[0] .. offsets[n] of the buffer, which a slice of a long column shares with the whole column;
    `first` = offsets[0] is the offset value of bytes[0], so the offsets index `bytes` shifted back by `first`."""
    import pyarrow as pa
    if isinstance(values, pa.ChunkedArray):
        values = values.combine_chunks()
    if not isinstance(values, pa.Array):
        values = pa.array(np.asarray(values, dtype=object).tolist(), type=pa.large_string())
    isz = 8 if pa.types.is_large_string(values.type) else 4
    n = len(values)
    validity, off_buf, data_buf = values.buffers()
    offsets = np.frombuffer(off_buf, dtype=np.int64 if isz == 8 else np.int32, count=n + 1, offset=values.offset * isz)
    first, last = int(offsets[0]), int(offsets[-1])
    data = np.frombuffer(data_buf, dtype=np.uint8)[first:last] if data_buf is not None and last > first else np.zeros(1, np.uint8)
    mask = None
    if values.null_count:
        lo = values.offset // 8  # unpack only the bytes of the rows in use: a chunk of a long column is a small slice of its bitmap
        bits = np.unpackbits(np.frombuffer(validity, dtype=np.uint8)[lo:(values.offset + n + 7) // 8], bitorder="little")
        bits = bits[values.offset - 8 * lo:values.offset - 8 * lo + n]
        mask = np.ascontiguousarray(1 - bits).astype(np.uint8)
    return offsets, isz, data, first, mask


def take_strings(index, values, thread_index=None):
    """b200_take_strings: the arrow string column `values` gathered by `index` -> (pyarrow large_string array with nulls where a row is
    missing, whether a row was missing).  Only the bytes of `values`' own rows are copied to the device.  With `thread_index` the
    gather runs on that worker's slot, after the work already queued there (filter compaction gathers by the kept rows it computed
    on that slot), and waits for that slot only; without it, on slot 0 after every slot and torch's stream."""
    import contextlib

    import pyarrow as pa
    torch = _torch()
    ctx = _lib.context()
    if thread_index is None:
        ctx.sync()
        slot, stream = 0, contextlib.nullcontext()
    else:
        slot = ctx.slot(thread_index)
        stream = torch.cuda.stream(torch.cuda.ExternalStream(ctx.stream(slot), device=f"cuda:{ctx.device}"))
    with stream:  # a slot's stream: the copies and temporaries are ordered with the gather, torch's cache reuses them after it
        idx = _staged_index(index)
        n = len(idx)
        offsets, isz, data, first, mask = _string_source(values)
        src_len = len(offsets) - 1
        d_off, d_data = _staged(offsets), _staged(data)
        d_mask = None if mask is None else _staged(mask)
        out_off = torch.empty(n + 1, dtype=torch.int64, device=idx.device)
        valid = torch.empty(max(n, 1), dtype=torch.uint8, device=idx.device)
        size, missing = C.c_int64(0), C.c_int32(0)
        if thread_index is None:
            torch.cuda.synchronize(idx.device)  # the staging copies run on torch's stream, the gather on a slot's
        # the device pointer the offsets index: the staged bytes start at offset value `first`
        args = (ctx._h, slot, idx.data_ptr(), idx.element_size(), n, d_off.data_ptr(), isz, d_data.data_ptr() - first,
                None if d_mask is None else d_mask.data_ptr(), src_len, out_off.data_ptr())
        _lib.check(_lib.lib().b200_take_strings(*args, None, valid.data_ptr(), 0, C.byref(size), C.byref(missing)))
        out_bytes = torch.empty(max(size.value, 1), dtype=torch.uint8, device=idx.device)
        if size.value:
            _lib.check(_lib.lib().b200_take_strings(*args, out_bytes.data_ptr(), valid.data_ptr(), size.value, C.byref(size), C.byref(missing)))
        valid = valid[:n].cpu().numpy()
        off_host, bytes_host = out_off.cpu().numpy(), out_bytes[:size.value].cpu().numpy()
    bitmap = pa.py_buffer(np.packbits(valid.astype(bool), bitorder="little")) if missing.value else None
    arr = pa.LargeStringArray.from_buffers(n, pa.py_buffer(off_host), pa.py_buffer(bytes_host), bitmap, int(n - valid.sum()) if missing.value else 0)
    return arr, bool(missing.value)


def _to_host(x):
    if _lib.is_device(x):
        _lib.context().sync()
        return _device_tensor(x).cpu().numpy()
    return np.asarray(x)


def gather(columns, index, src_len, device):
    """{name: column} gathered by `index`: fixed-width columns through b200_take (16 per launch), strings through b200_take_strings.
    `device(column)` says where a fixed-width result goes.  A column with a missing row, or one that was masked, is a host np.ma."""
    out = {}
    fixed = []
    for name, col in columns.items():
        if _hash.is_string_column(col):
            out[name] = take_strings(index, col)[0]
            continue
        data, mask = _lib.split_mask(col)
        fixed.append((name, data, mask, device(col)))
        out[name] = None
    for dev in (False, True):
        group = [f for f in fixed if f[3] == dev]
        if not group:
            continue
        for (name, _, mask, _), (values, valid) in zip(group, take(index, [(d, m) for _, d, m, _ in group], src_len, dev)):
            if valid is None and mask is None:
                out[name] = values
            else:
                values = _to_host(values)
                out[name] = np.ma.array(values, mask=np.zeros(len(values), bool) if valid is None else _to_host(valid) == 0)
    return out


# ---- the frame pieces ---------------------------------------------------------------------------------------------------------
def _concat(a, b):
    if _hash.is_string_column(a) or _hash.is_string_column(b):
        import pyarrow as pa

        def large(x):
            x = x if isinstance(x, pa.Array) else pa.array(np.asarray(x, dtype=object).tolist(), type=pa.large_string())
            return x if pa.types.is_large_string(x.type) else x.cast(pa.large_string())
        return pa.concat_arrays([large(a), large(b)])
    if _lib.is_device(a) and _lib.is_device(b):
        return _torch().cat([_device_tensor(a), _device_tensor(b)])
    if np.ma.isMaskedArray(a) or np.ma.isMaskedArray(b):
        return np.ma.concatenate([np.ma.asarray(_to_host(a) if _lib.is_device(a) else a), np.ma.asarray(b)])
    return np.concatenate([_to_host(a), _to_host(b)])


def _materialize(frame, name):
    """a virtual column's values over the whole frame (unfiltered), on the device when the frame's columns are"""
    values = frame.evaluate(name)
    col = frame.columns[name]
    if col.columns and _lib.on_device(col) and values.dtype.kind not in "mM":
        return _torch().from_numpy(values).to(f"cuda:{_lib.context().device}")
    return values


def extract(frame):
    """DataFrame.extract (join.py:160): the frame's rows that pass its filter, virtual columns evaluated, as a Frame without a filter"""
    from .frame import Frame
    columns = {name: _materialize(frame, name) if _is_virtual(col) else col for name, col in frame.columns.items()}
    if frame._filter is None:
        return Frame(columns, executor=frame.executor, variables=frame.variables)
    rows = np.flatnonzero(frame.evaluate(frame._filter_expression))
    columns = gather(columns, rows, frame.length, _lib.is_device)
    return Frame(columns, executor=frame.executor, variables=frame.variables)


def index(frame, expression, nmaps=None):
    """DataFrame._index (vaex/dataframe.py:514-572): the device index_hash of `expression` over the frame's rows (its filter is not
    applied: the join extracts the right side first)"""
    columns = frame._with_columns([expression]).columns  # an expression key is evaluated on the device like GroupBy's keys
    dtype = _lib.dtype_of(columns[expression])
    try:
        part = taskpart.TaskPartIndex(expression, dtype, nmaps or frame.executor.nthreads)
    except TypeError as e:
        if dtype.kind in "OUS" or _hash.is_string_column(columns[expression]):
            raise TypeError(f"cannot join on the string key {expression!r}: index_hash_string, the device index for string keys, "
                            "is not available") from e
        raise
    frame.executor.execute(columns, [execution.Task(part)], frame.length)
    return part.index


def _rename_in(text, old, new):
    """rename the name `old` to `new` in an expression's text"""
    import ast

    class Sub(ast.NodeTransformer):
        def visit_Name(self, node):
            if node.id == old:
                node.id = new
            return node
    return ast.unparse(Sub().visit(ast.parse(text, mode="eval")))


def join(df, other, on=None, left_on=None, right_on=None, lprefix='', rprefix='', lsuffix='', rsuffix='', how='left', allow_duplication=False,
         prime_growth=False, cardinality_other=None, inplace=False):
    """DataFrameLocal.join (vaex/join.py:125-297).  `prime_growth` and `cardinality_other` only tune the CPU table and are ignored."""
    from .frame import Frame
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
    on, left_on, right_on = (None if x is None else str(x) for x in (on, left_on, right_on))
    left_on = left_on or on
    right_on = right_on or on
    for name in right.columns:
        if left_on and (rprefix + name + rsuffix == lprefix + left_on + lsuffix):
            continue  # it's ok when we join on the same column name
        if name in left.columns and rprefix + name + rsuffix == lprefix + name + lsuffix:
            raise ValueError('column name collision: {} exists in both column, and no proper suffix given'.format(name))

    right = extract(right)
    N = left.length
    n_other = len(right)
    real = {k: v for k, v in left.columns.items() if not _is_virtual(v)}
    virtual = {k: v.expression for k, v in left.columns.items() if _is_virtual(v)}
    lfilter = left._filter_expression
    lookup = None
    lookup_device = False
    if left_on is not None or right_on is not None:
        ix = index(right, right_on)
        duplicates_right = ix.has_duplicates
        if duplicates_right and not allow_duplication:
            raise ValueError('This join will lead to duplication of rows which is disabled, pass allow_duplication=True')
        lookup_dtype = required_dtype_for_max(n_other)
        columns = left._with_columns([left_on]).columns
        key = columns[left_on]
        lookup_device = _lib.on_device(key) and not (_is_virtual(key) and not key.columns)  # a key without inputs is looked up on the host
        if lookup_device:
            torch = _torch()
            lookup = torch.full((N,), int(np.iinfo(lookup_dtype).max), dtype=_torch_dtype(lookup_dtype), device=f"cuda:{_lib.context().device}")
            torch.cuda.synchronize(lookup.device)  # the fill runs on torch's stream, map_index writes on a slot's
        else:
            lookup = np.full(N, np.iinfo(lookup_dtype).max, dtype=lookup_dtype)
        part = taskpart.TaskPartLookup(ix, left_on, lookup, duplicates_right)
        left.executor.execute(columns, [execution.Task(part)], N)  # every row, filtered or not (join.py:209 ignore_filter=True)
        _, extra = part.get_result()
        if extra:
            # the right's duplicates: the left's rows repeated, ordered by (left row, right row), and their right rows (join.py:210-215)
            torch = _torch()
            lookup_left = torch.cat([e[1] for e in extra])
            lookup_right = torch.cat([e[2] for e in extra])
            if not lookup_device:
                lookup_left, lookup_right = lookup_left.cpu().numpy(), lookup_right.cpu().numpy()
            repeated = gather(real, lookup_left, N, _lib.is_device)
            real = {k: _concat(v, repeated[k]) for k, v in real.items()}
            lookup = torch.cat([lookup.to(torch.int64), lookup_right]) if lookup_device else np.concatenate([lookup.astype(np.int64), lookup_right])
        if inner:
            from . import expression as _expr
            total = len(lookup)
            if lookup_device:
                torch = _torch()
                keep = (lookup != -1).to(torch.uint8)
                rows = torch.arange(total, dtype=torch.int64, device=lookup.device)
            else:
                keep = (lookup != -1).view(np.uint8)
                rows = np.arange(total, dtype=np.int64)
            if lookup_device:
                torch.cuda.synchronize(lookup.device)
            kept, (rows, lookup) = _expr.compact(0, keep, [rows, lookup])
            rows, lookup = _device_tensor(rows)[:kept].clone(), _device_tensor(lookup)[:kept].clone()
            if not lookup_device:
                rows, lookup = rows.cpu().numpy(), lookup.cpu().numpy()
            real = gather(real, rows, total, _lib.is_device)

    # renaming, so all names are unique (join.py:231-255)
    right_cols = dict(right.columns)
    right_names = list(right_cols)
    left_names = list(real) + list(virtual)

    def rename_left(old, new):
        nonlocal lfilter
        if old == new:
            return
        if old in real:
            real[new] = real.pop(old)
        else:
            virtual[new] = virtual.pop(old)
        for k in list(virtual):
            virtual[k] = _rename_in(virtual[k], old, new)
        if lfilter is not None:
            lfilter = _rename_in(lfilter, old, new)
    for name in list(right_names):
        if name in left_names:
            all_names = list(set(right_names + left_names))
            all_names.append(mangle_name(lprefix, name, lsuffix))
            all_names.remove(name)
            new_name = mangle_name(rprefix, name, rsuffix)
            if new_name != left_on:
                if new_name in all_names:
                    new_name = find_valid_name(new_name, all_names)
                right_cols = {(new_name if k == name else k): v for k, v in right_cols.items()}
                right_names[right_names.index(name)] = new_name
            all_names = list(set(right_names + left_names))
            all_names.remove(name)
            new_name = mangle_name(lprefix, name, lsuffix)
            if new_name in all_names:
                new_name = find_valid_name(new_name, all_names)
            rename_left(name, new_name)
            left_names[left_names.index(name)] = new_name

    variables = dict(left.variables)
    variables.update(right.variables)
    added = {}
    for name, col in right_cols.items():
        if name == left_on and name in left_names:
            continue  # the join column is not added twice
        assert name not in left_names
        added[name] = col
    if added:
        if lookup is None:
            if n_other != N:
                raise ValueError(f"a join without a key needs equal row counts: {N} rows on the left, {n_other} on the right")
        else:
            added = gather(added, lookup, n_other, lambda col: lookup_device)
    columns = dict(real)
    columns.update(added)
    result = Frame(columns, executor=left.executor, categories=left.categories, variables=variables)
    for name, text in virtual.items():
        result.add_virtual_column(name, text)
    if lfilter is not None:
        result = result.filter(lfilter)
    if inplace:
        df.__dict__.update(result.__dict__)
        return df
    return result
