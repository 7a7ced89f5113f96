"""Frame.sort (vaex/dataframe.py:4694-4745) and Frame.take (vaex/dataframe.py:4444-4481) with the argsort on the device.

The reference builds an arrow table of the `by` columns over the filtered rows and runs ``pa.compute.sort_indices`` on the host;
here every key is staged to the device once (device columns in place, host columns copied, expression keys evaluated on the
device, string keys replaced by their rank in a device string set), a filtered frame's keys are compacted with ``b200_compact``
together with their row numbers, and ``b200_argsort`` (csrc/sort.cu) returns the permutation.  The rows are then gathered with
``join.gather``: device columns stay on the device, host columns come back to the host, strings as arrow, masks kept.

Arrow's conversion of the keys is kept: a masked value is null, a float NaN stays NaN, and NaT is null in a datetime column
without a mask while in a masked one only the mask decides (an unmasked NaT is the value INT64_MIN, ``pa.array(np.ma...)``).
"""
import ctypes as C

import numpy as np

from . import _lib
from . import hash as _hash
from . import join as _join

MAX_ROWS = 2 ** 32 - 1  # B200_SORT_MAX_ROWS: the radix scatter's positions are 32-bit
MAX_KEYS = 16           # B200_SORT_MAX_KEYS
HIST_BYTES = 256 * 4 * 4096 + 512  # radix histograms (at most 256 counters x ~2048 blocks) and the AND / OR pair, rounded up


def scratch_bytes(nrows):
    """device bytes one sort of `nrows` rows needs: the int64 permutation (torch) and the library's scratch (two 64-bit words and
    one 64-bit payload per row, csrc/sort.cu)"""
    return 8 * nrows + 24 * nrows + HIST_BYTES


def free_bytes(device):
    """device memory a sort may take: free on the device, held idle by the context's block cache or by torch's allocator"""
    import torch
    free, _ = torch.cuda.mem_get_info(device)
    cached = _lib.context(device).mem_stats()["cached"]
    return free + cached + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


def _issequence(x):
    return isinstance(x, (tuple, list, np.ndarray))


def normalize(by, ascending):
    """by / ascending as the reference reads them (:4724-4733): lists of equal length, a key ascending only when its flag `is True`"""
    by = [str(b) for b in (by if _issequence(by) else [by])]
    if isinstance(ascending, list):
        if len(ascending) != len(by):
            raise AssertionError('If "ascending" is a list, it must have the same number of elements as "by".')
    else:
        ascending = list(ascending if _issequence(ascending) else [ascending]) * len(by)
    return by, [a is True for a in ascending]


class Key:
    """one key staged for b200_argsort: device data (any dtype of its width), its b200_dtype, byte order, device null mask"""
    __slots__ = ("data", "code", "byteswap", "mask", "descending", "nat_is_null")

    def __init__(self, data, code, byteswap=False, mask=None, descending=False, nat_is_null=False):
        self.data, self.code, self.byteswap, self.mask = data, code, bool(byteswap), mask
        self.descending, self.nat_is_null = bool(descending), bool(nat_is_null)


def _code(dtype):
    dtype = np.dtype(dtype)
    if dtype.kind in "mM":
        return _lib.I64  # signed: dates before 1970 and NaT (INT64_MIN) order as arrow's int64 timestamps do
    return _lib.DTYPE_CODE[dtype.newbyteorder("=").name]


def _upload(a):
    """a host array's bytes as a device array of the same width (byte order kept: the encode kernel swaps)"""
    import torch
    from .expression import DeviceArray
    a = np.ascontiguousarray(a)
    t = torch.from_numpy(a.view(np.uint8)).to(f"cuda:{_lib.context().device}")
    return DeviceArray(t.data_ptr(), len(a), f"u{a.dtype.itemsize}", keep=t)


def stage_key(col, nrows, descending):
    """a frame column -> Key over its nrows (unfiltered) rows"""
    if _hash.is_string_column(col):
        # arrow's bytewise order: the rank of each string among the distinct ones (device string set, the host sorts only the
        # distinct strings); the set is sorted in the key's own direction with null last, so the ranks sort ascending
        hm = _hash.HashMapUnique(np.dtype("O"), nmaps=1)
        hm.add(col)
        ranks = hm.sorted(ascending=not descending)._internal.map_ordinal(col, device=True)
        return Key(ranks, _lib.I64)
    if getattr(col, "device_virtual", False):
        return Key(col.chunk(0, 0, nrows), _code(col.dtype), descending=descending)
    if _lib.is_device(col):
        return Key(col, _code(_lib.dtype_of(col)), descending=descending)
    data, mask = _lib.split_mask(col)
    data = np.asarray(data)
    return Key(_upload(data), _code(data.dtype), not data.dtype.isnative, None if mask is None else _upload(mask.view(np.uint8)), descending,
               nat_is_null=data.dtype.kind in "mM" and mask is None)


def argsort(keys, nrows):
    """b200_argsort over staged keys of `nrows` rows -> the stable permutation (device int64 tensor)"""
    import torch
    if nrows > MAX_ROWS:
        raise ValueError(f"sort: {nrows} rows exceed the limit of {MAX_ROWS} rows of one device sort (32-bit scatter positions)")
    if not 1 <= len(keys) <= MAX_KEYS:
        raise ValueError(f"sort: between 1 and {MAX_KEYS} keys are supported, got {len(keys)}")
    ctx = _lib.context()
    need, free = scratch_bytes(nrows), free_bytes(ctx.device)
    if need > free:
        raise MemoryError(f"sort of {nrows} rows: the permutation and the radix scratch ({need} bytes) exceed the {free} bytes free on the device")
    perm = torch.empty(nrows, dtype=torch.int64, device=f"cuda:{ctx.device}")
    arr = (_lib.SortKey * len(keys))()
    for a, k in zip(arr, keys):
        a.data, a.dtype, a.byteswap = _lib.column(k.data).ptr, k.code, int(k.byteswap)
        a.mask = None if k.mask is None else _lib.column(k.mask).ptr
        a.descending, a.nat_is_null = int(k.descending), int(k.nat_is_null)
    torch.cuda.synchronize(perm.device)  # staging copies run on torch's stream
    ctx.sync()                           # device expressions, string ranks and compaction on the slots' streams
    _lib.check(_lib.lib().b200_argsort(ctx._h, 0, len(keys), arr, nrows, perm.data_ptr(), 0))
    return perm


def _compact(keep, columns):
    """b200_compact of device / host columns by a keep mask, 16 columns per call -> (rows kept, [device arrays])"""
    from .expression import compact
    kept, out = 0, []
    for i in range(0, len(columns), 16):
        kept, part = compact(0, keep, columns[i:i + 16])
        out += part
    return kept, out


def filtered_rows(frame, keys=()):
    """the unfiltered row numbers of a filtered frame's rows (device int64) and the keys compacted to those rows alongside"""
    import torch
    n = frame.length
    keep = frame._filter.chunk(0, 0, n)
    rows = torch.arange(n, dtype=torch.int64, device=f"cuda:{_lib.context().device}")
    torch.cuda.synchronize(rows.device)
    cols = [rows] + [k.data for k in keys] + [k.mask for k in keys if k.mask is not None]
    kept, out = _compact(keep, cols)
    rows, datas, masks = out[0], out[1:1 + len(keys)], iter(out[1 + len(keys):])
    staged = [Key(d, k.code, k.byteswap, None if k.mask is None else next(masks), k.descending, k.nat_is_null) for d, k in zip(datas, keys)]
    return kept, rows, staged


def sorted_rows(frame, by, ascending):
    """the unfiltered row numbers of the frame's filtered rows in sorted order (device int64), None when no row passes"""
    if frame.length == 0:
        return None
    f = frame._with_columns(by)
    keys = [stage_key(f.columns[name], f.length, not asc) for name, asc in zip(by, ascending)]
    if f._filter is None:
        return argsort(keys, f.length)
    kept, rows, keys = filtered_rows(f, keys)
    if kept == 0:
        return None
    perm = argsort(keys, kept)
    return _join.take(perm, [(rows, None)], kept, True)[0][0]


def take_index(frame, indices, filtered):
    """Frame.take's indices -> int64 unfiltered row numbers (host numpy or device tensor).  An index outside [0, n) raises
    IndexError before anything is gathered, where numpy's fancy indexing in the reference would wrap a negative one."""
    if _lib.is_device(indices):
        import torch
        idx = _join._device_tensor(indices)
        if idx.dtype == torch.uint64:
            idx = idx.view(torch.int64)  # >= 2^63 turns negative: out of range either way
        elif idx.dtype in (torch.uint8, torch.uint16, torch.uint32):
            idx = idx.to(torch.int64)
        elif idx.dtype not in (torch.int8, torch.int16, torch.int32, torch.int64):
            raise TypeError(f"take: indices must be integers, not {idx.dtype}")
        lo, hi = (int(idx.min()), int(idx.max())) if len(idx) else (0, -1)
    else:
        idx = np.asarray(indices)
        if idx.size == 0:
            idx = idx.astype(np.int64)
        if idx.ndim != 1 or idx.dtype.kind not in "iu":
            raise TypeError(f"take: indices must be a 1-d sequence of integers, not {idx.dtype}")
        lo, hi = (int(idx.min()), int(idx.max())) if len(idx) else (0, -1)
        if idx.dtype.kind == "u":
            idx = idx.astype(np.int64) if hi <= np.iinfo(np.int64).max else idx
        if not idx.dtype.isnative:
            idx = idx.astype(idx.dtype.newbyteorder("="))
    rows = None
    bound = frame.length
    if filtered and frame._filter is not None:
        bound, rows, _ = filtered_rows(frame)
    if lo < 0 or hi >= bound:
        raise IndexError(f"take: index {lo if lo < 0 else hi} is out of bounds for {bound} rows")
    if rows is None:
        return idx
    return _join.take(idx, [(rows, None)], bound, True)[0][0]
