"""``HashMapUnique`` — host-side mirror of vaex.hash.HashMapUnique over the device ordered_set.

Reference: packages/vaex-core/vaex/hash.py:62-292 (add / merge / flatten / keys / map / isin / sorted / limit and the
null/nan bookkeeping).  String and object keys are out of scope (SURVEY.md 8f row 3)."""
import numpy as np

from . import _lib, superutils


def is_string_column(ar):
    """pyarrow string / large_string arrays, numpy object / unicode arrays"""
    try:
        import pyarrow as pa
        if isinstance(ar, (pa.Array, pa.ChunkedArray)):
            return pa.types.is_string(ar.type) or pa.types.is_large_string(ar.type)
    except ImportError:  # pragma: no cover
        pass
    return isinstance(ar, np.ndarray) and ar.dtype.kind in "OU"


def ordered_set_type_from_dtype(dtype):
    dtype = np.dtype(dtype)
    if dtype.kind in "OU":  # vaex.hash: string keys -> ordered_set_string (src/hash_string.hpp)
        return superutils.ordered_set_string
    if dtype.kind in "mM":
        dtype = np.dtype("int64")
    name = "ordered_set_" + dtype.newbyteorder("=").name
    if not hasattr(superutils, name):
        raise ValueError(f"Could not find a class ({name}), seems {dtype} is not supported.")
    return getattr(superutils, name)


def index_type_from_dtype(dtype, transient=True, prime_growth=False):
    """vaex.hash.index_type_from_dtype (vaex/hash.py:56-60, vaex/utils.py:754-790 with support_non_native=False): the index_hash
    class for a key dtype; datetimes and timedeltas are indexed as int64, and a byte-swapped dtype has no class (big-endian float64
    excepted, which the reference maps to float64).  ``transient`` and ``prime_growth`` only choose the CPU table's string storage
    and growth policy, so they change nothing here.  String keys have no device index yet."""
    if str(dtype) == "string" or np.dtype(dtype).kind in "OUS":
        raise TypeError(f"no index_hash for dtype {dtype}: string keys are not indexed on the device")
    dtype = np.dtype(dtype)
    name = "float64" if str(dtype) == ">f8" else "int64" if dtype.kind in "mM" else str(dtype)
    if not hasattr(superutils, "index_hash_" + name):
        raise ValueError(f"Could not find a class (index_hash_{name}), seems {dtype} is not supported.")
    return getattr(superutils, "index_hash_" + name)


class HashMapUnique:
    """HashMap that maps keys to unique integers (vaex/hash.py:62-64)."""

    def __init__(self, dtype, nmaps=1, limit=None, _internal=None):
        self.dtype = np.dtype(dtype)
        self.dtype_item = self.dtype
        limit = -1 if limit is None else limit
        if _internal is None:
            self._internal = ordered_set_type_from_dtype(self.dtype)(nmaps, limit)
        else:
            self._internal = _internal

    @property
    def is_string(self):
        return self.dtype.kind in "OU"

    def flatten(self):
        # vaex/hash.py:75-80: rebuild a 1-shard set from key_array() so ordinals become global
        if self.is_string:  # the device string set already answers map_ordinal with GLOBAL ordinals (local + offsets[shard])
            return self
        keys = self._internal.key_array()
        m = type(self._internal)(keys, self.null_index, self.nan_count, self.null_count, self.fingerprint)
        return HashMapUnique(self.dtype, _internal=m)

    @classmethod
    def from_keys(cls, keys, dtype=None, fingerprint=""):
        # vaex/hash.py:112-150
        dtype = np.dtype(keys.dtype if dtype is None else dtype)
        null_count, null_index = 0, -1
        if np.ma.isMaskedArray(keys):
            null_count = int(keys.mask.sum())
            if null_count == 1:
                null_index = int(np.where(np.ma.getmaskarray(keys))[0][0])
            elif null_count > 1:
                raise ValueError("key arrays contained more than 1 null value")
            keys = keys.data
        keys = np.asarray(keys)
        nancount = int(np.isnan(keys).sum()) if dtype.kind == "f" else 0
        internal = ordered_set_type_from_dtype(dtype)(keys, null_index, nancount, null_count, fingerprint)
        return cls(dtype, _internal=internal)

    def add(self, ar, return_inverse=False):
        # vaex/hash.py:152-171
        chunk_size = 1024 * 1024
        if self.is_string:
            return self._internal.update(ar, -1, chunk_size=chunk_size, bucket_size=chunk_size * 4, return_values=return_inverse)
        data, mask = _lib.split_mask(ar)
        if mask is not None:
            return self._internal.update(data, mask, -1, chunk_size=chunk_size, bucket_size=chunk_size * 4, return_values=return_inverse)
        if not _lib.is_device(ar):
            ar = np.ascontiguousarray(ar)
        return self._internal.update(ar, -1, chunk_size=chunk_size, bucket_size=chunk_size * 4, return_values=return_inverse)

    def __len__(self):
        return len(self._internal)

    def merge(self, others):
        self._internal.merge([getattr(o, "_internal", o) for o in others])

    def keys(self, mask=True):
        # vaex/hash.py:179-191
        ar = self._internal.key_array()
        if self.is_string:
            return np.array(ar.to_pylist(), dtype=object)
        if self.dtype_item.kind in "mM":
            ar = ar.view(self.dtype_item)
        if mask and self.has_null:
            m = np.zeros(ar.shape, dtype="?")
            m[self.null_index] = 1
            ar = np.ma.array(ar, mask=m)
        return ar

    def map(self, keys, check_missing=False):
        """Map key values to unique integers (vaex/hash.py:193-214)."""
        if self.is_string:
            indices = self._internal.map_ordinal(keys)
            return np.ma.array(indices, mask=indices == -1) if check_missing else indices
        masked = isinstance(keys, np.ndarray) and np.ma.isMaskedArray(keys)
        data = np.ascontiguousarray(keys.data) if masked else keys
        indices = self._internal.map_ordinal(data)
        if masked:
            m = np.ma.getmaskarray(keys)
            if self.null_index > np.iinfo(indices.dtype).max:
                indices[m] = -1
            else:
                indices[m] = self.null_index
        if check_missing:
            indices = np.ma.array(indices, mask=indices == -1)
        return indices

    def isin(self, values):
        if isinstance(values, np.ndarray) and np.ma.isMaskedArray(values):
            isin = self._internal.isin(np.ascontiguousarray(values.data))
            isin[np.ma.getmaskarray(values)] = False
            return isin
        return self._internal.isin(values)

    has_null = property(lambda self: self._internal.has_null)
    has_nan = property(lambda self: self._internal.has_nan)
    null_index = property(lambda self: self._internal.null_index)
    nan_index = property(lambda self: self._internal.nan_index)
    nan_count = property(lambda self: self._internal.nan_count)
    null_count = property(lambda self: self._internal.null_count)

    @property
    def fingerprint(self):
        return self._internal.fingerprint

    def sorted(self, ascending=True, return_keys=False):
        if self.is_string:
            return self._sorted_strings(ascending, return_keys)
        return self._sorted(ascending, return_keys)

    def _sorted_strings(self, ascending=True, return_keys=False):
        # vaex/hash.py:246-268 for string keys: arrow's (bytewise) order, the null key last; the sorted keys go into a fresh 1-shard
        # device set in that order, so ordinal == rank
        import pyarrow as pa
        import pyarrow.compute as pc
        keys = self._internal.key_array()
        valid = pc.drop_null(keys)
        sorted_keys = valid.take(pc.array_sort_indices(valid, order="ascending" if ascending else "descending"))
        if self.has_null:
            sorted_keys = pa.concat_arrays([sorted_keys, pa.array([None], type=sorted_keys.type)])
        internal = type(self._internal)(1)
        if len(sorted_keys):
            internal.update(sorted_keys)
        out = HashMapUnique(self.dtype, _internal=internal)
        return (out, np.array(sorted_keys.to_pylist(), dtype=object)) if return_keys else out

    def _sorted(self, ascending=True, return_keys=False):
        # vaex/hash.py:246-268 — arrow sorts nulls last; NaN sorts after every number
        keys = self.keys(mask=False)
        has_null = self.has_null
        idx = np.arange(len(keys))
        if has_null:
            idx = idx[idx != self.null_index]
        k = keys[idx]
        order = np.argsort(k, kind="stable")
        if not ascending:
            if k.dtype.kind == "f":
                nan = np.isnan(k[order])
                order = np.concatenate([order[~nan][::-1], order[nan]])
            else:
                order = order[::-1]
        sorted_keys = k[order]
        null_index = -1
        if has_null:
            sorted_keys = np.concatenate([sorted_keys, keys[self.null_index:self.null_index + 1]])
            null_index = len(sorted_keys) - 1
        internal = type(self._internal)(sorted_keys, null_index, self._internal.nan_count, self._internal.null_count, self.fingerprint + "-sorted")
        out = HashMapUnique(self.dtype, _internal=internal)
        return (out, sorted_keys) if return_keys else out

    def limit(self, limit):
        # vaex/hash.py:270-289
        keys = self.keys(mask=False)[:limit]
        null_index, null_count = self.null_index, 1
        if null_index >= limit or not self.has_null:
            null_index, null_count = -1, 0
        nan_count = int(np.isnan(keys).sum()) if self.dtype_item.kind == "f" else 0
        internal = type(self._internal)(keys, null_index, nan_count, null_count, self.fingerprint + f"-limit-{limit}")
        return HashMapUnique(self.dtype, _internal=internal)

    def __sizeof__(self):
        return self._internal.__sizeof__()


class CombinedCodes:
    """The combined group code of a sparse multi-key groupby as a virtual int64 column that is evaluated ON THE DEVICE, chunk
    by chunk, inside the executor's feed loop — the reference builds it as the expression
    ``sum_k _ordinal_values(key_k, hash_map_k).astype(...) * cumulative_counts[k+1]`` (vaex/groupby.py:555-566,
    vaex/functions.py:2454-2463) and evaluates it with numpy per chunk.

    ``chunk(thread_index, i1, i2)`` runs one fused lookup kernel (``b200_set_combine``) on the slot of that executor thread
    and returns a device array; the task part that consumes it runs on the same slot, i.e. the same CUDA stream."""

    device_virtual = True  # the executor calls chunk(thread_index, i1, i2) instead of slicing

    def __init__(self, columns, hash_maps, multipliers):
        if not 1 <= len(columns) <= 8:
            raise ValueError("between 1 and 8 key columns can be combined")
        assert len(columns) == len(hash_maps) == len(multipliers)
        self.columns = list(columns)
        self.hash_maps = list(hash_maps)
        self.multipliers = [int(m) for m in multipliers]
        self.dtype = np.dtype("int64")
        self._ctx_cached = None
        self._buffers = {}

    def __len__(self):
        return len(self.columns[0])

    @property
    def _ctx(self):
        if self._ctx_cached is None:
            self._ctx_cached = _lib.context()
        return self._ctx_cached

    def _buffer(self, thread_index, n):
        import torch
        buf = self._buffers.get(thread_index)
        if buf is None or buf.numel() < n:
            buf = torch.empty(max(n, 1), dtype=torch.int64, device=f"cuda:{self._ctx.device}")
            self._buffers[thread_index] = buf
        return buf[:n]

    def chunk(self, thread_index, i1, i2):
        import ctypes as C
        n = i2 - i1
        out = self._buffer(thread_index, n)
        if n == 0:
            return out
        nk = len(self.columns)
        keep, kptr, mptr = [], (C.c_void_p * nk)(), (C.c_void_p * nk)()
        for k, col in enumerate(self.columns):
            # a previous stage's codes (vaex/groupby.py:572-582) are produced on this worker's slot, like every device-virtual column
            part = _lib.chunk_of(col, thread_index, i1, i2)
            mask = None
            if isinstance(part, np.ndarray) and np.ma.isMaskedArray(part):
                mask = np.ma.getmaskarray(part)
                part = part.data
            if isinstance(part, np.ndarray) and not part.dtype.isnative:
                part = part.astype(part.dtype.newbyteorder("="))
            c = _lib.column(part)
            if c.dtype.itemsize != self.hash_maps[k].dtype.itemsize:
                raise RuntimeError("stride not equal to bytesize for key values")
            keep.append(c)
            kptr[k] = c.ptr
            if mask is not None:
                m = _lib.mask_column(mask)
                keep.append(m)
                mptr[k] = m.ptr
        sets = (C.c_void_p * nk)(*[hm._internal._h for hm in self.hash_maps])
        mult = (C.c_int64 * nk)(*self.multipliers)
        _lib.check(_lib.lib().b200_set_combine(self._ctx._h, self._ctx.slot(thread_index), nk, sets, kptr, mptr, mult, n, out.data_ptr(),
                                               _lib.memspace(*keep), 0))
        return out

    def decode(self, codes):
        """group code -> ordinal of every parent key (the div/mod chain of GrouperCombined, vaex/groupby.py:352-358)"""
        codes = np.asarray(codes, dtype=np.int64)
        out, left = [], codes
        for m in self.multipliers:
            out.append(left // m)
            left = left % m
        return out


class StringCodes:
    """``_ordinal_values(key, hash_map_unique)`` for a STRING key column as a device-evaluated int64 column: every chunk's strings
    are probed against the device string set on the worker's slot (vaex/functions.py:2454-2463 + HashMapUnique.map,
    vaex/hash.py:193-214); the codes feed a BinnerOrdinal exactly like the reference's pass 2 does (vaex/groupby.py:303-317)."""

    device_virtual = True

    def __init__(self, column, hash_map):
        self.columns = [column]  # host strings: the executor feeds host chunks
        self.hash_map = hash_map
        self.dtype = np.dtype("int64")

    def __len__(self):
        return len(self.columns[0])

    def chunk(self, thread_index, i1, i2):
        return self.hash_map._internal.map_ordinal(self.columns[0][i1:i2], slot=thread_index, device=True)
