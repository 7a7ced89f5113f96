"""Drop-in mirror of the ordinal-encoder part of ``vaex.superutils``: ``ordered_set_<dtype>`` and ``hash``.

Reference: packages/vaex-core/src/hash_primitives.cpp:3-25, 45-56 (bindings), src/hash_primitives.hpp:437-725 (ordered_set),
src/superutils.cpp:265 (``hash``).  Same constructor overloads, method names, keyword arguments, return dtypes and error
messages.  Keys may be numpy arrays (host, staged per call) or device arrays (``__cuda_array_interface__``).

Ordinals are identical to the reference run sequentially with chunks in order (one ``update`` call per chunk).  With more
than one thread the reference's own ordinals are timing dependent (insertion order under per-shard mutexes); the device
version always returns the sequential answer.
"""
import copyreg
import ctypes as C
import math

import numpy as np

from . import _lib


def hash(x):
    """``vaex.superutils.hash`` — splitmix64 finaliser (src/hash.hpp:40-45)."""
    return _lib.lib().b200_hash64(int(x) & 0xFFFFFFFFFFFFFFFF)


class _OrderedSet:
    _dtype = None
    _code = None

    def __init__(self, *args, **kwargs):
        self._ctx = _lib.context()
        self._h = C.c_void_p()
        self.fingerprint = ""
        self.sealed = False
        first = args[0] if args else kwargs.get("nmaps", 1)
        if isinstance(first, (int, np.integer)) and not isinstance(first, bool):
            nmaps = int(first)
            limit = int(args[1]) if len(args) > 1 else int(kwargs.get("limit", -1))
            self.nmaps = nmaps
            _lib.check(_lib.lib().b200_set_create(self._ctx._h, self._code, nmaps, limit, C.byref(self._h)))
        else:
            # ordered_set_<T>(keys, null_index, nan_count, null_count, fingerprint)  (src/hash_primitives.hpp:486-537)
            keys, null_index, nan_count, null_count = args[0], int(args[1]), int(args[2]), int(args[3])
            self.fingerprint = args[4] if len(args) > 4 else ""
            keys = np.ascontiguousarray(np.asarray(keys), dtype=self._np_dtype())
            if keys.ndim != 1:
                raise RuntimeError("Expected a 1d array")
            self.nmaps = 1
            _lib.check(_lib.lib().b200_set_from_keys(self._ctx._h, self._code, keys.ctypes.data if keys.size else None, len(keys), null_index, nan_count,
                                                     null_count, C.byref(self._h)))
            self.sealed = True

    @classmethod
    def _np_dtype(cls):
        return np.dtype(cls._dtype)

    def _key_column(self, values):
        """Key values as a column of the set's own dtype.  The reference takes keys as ``py::array_t<T>``
        (src/hash_primitives.hpp:72,81,539,611), whose default forcecast converts a host array of another dtype or byte order by
        VALUE (``update(np.array([1.7, 2.2]))`` on an int64 set inserts 1 and 2; a big-endian column inserts its numbers, not its
        swapped bytes); host arrays get the same conversion here.  Device columns are read in place, so they must already hold
        the set's dtype: only same-width integer types (whose bits are their values) are accepted in its stead."""
        native = self._np_dtype()
        cai = getattr(values, "__cuda_array_interface__", None)
        if cai is not None and not isinstance(values, np.ndarray):
            col = _lib.column(values)
            dt = col.dtype
            same_bits = dt.isnative and dt.itemsize == native.itemsize and dt.kind in "biumM" and native.kind in "biu"
            if dt != native and not same_bits:
                raise TypeError(f"{type(self).__name__}: a device column of dtype {dt} cannot be read as {native} keys; convert it first")
            return col
        a = np.asarray(values)
        if a.dtype != native:
            with np.errstate(invalid="ignore", over="ignore"):
                a = a.astype(native)
        return _lib.column(a)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().b200_set_destroy(h)
            except Exception:
                pass
            self._h = None

    # -- reference protocol --------------------------------------------------------------------------
    def update(self, values, *args, **kwargs):
        """update(values[, masks], start_index=0, chunk_size=..., bucket_size=..., return_values=False)"""
        names = ["start_index", "chunk_size", "bucket_size", "return_values"]
        masks = kwargs.pop("masks", None)
        args = list(args)
        if args and not isinstance(args[0], (int, np.integer, bool)):
            masks = args.pop(0)
        opts = dict(start_index=0, chunk_size=1024 * 128, bucket_size=1024 * 128, return_values=False)
        for n, v in zip(names, args):
            opts[n] = v
        opts.update(kwargs)
        if opts["bucket_size"] < opts["chunk_size"]:
            raise RuntimeError("bucket size should be larger than chunk_size")
        col = self._key_column(values)
        mcol = None
        if masks is not None:
            mcol = _lib.mask_column(masks)
            if mcol.length != col.length:
                raise RuntimeError("array and mask should be of same size")
        n = col.length
        rv = bool(opts["return_values"])
        out_values = np.empty(n if rv else 1, np.int64)
        out_map = np.empty(n if rv else 1, np.int16)
        _lib.check(_lib.lib().b200_set_update(self._h, 0, col.ptr, None if mcol is None else mcol.ptr, n, int(opts["start_index"]), int(rv),
                                              out_values.ctypes.data, out_map.ctypes.data, _lib.memspace(col, mcol), 0))
        if rv:
            return out_values, out_map
        return None

    def merge(self, others):
        if self.sealed:
            raise RuntimeError("hashmap is sealed, cannot merge")
        if not others:
            return
        arr = (C.c_void_p * len(others))(*[o._h for o in others])
        _lib.check(_lib.lib().b200_set_merge(self._h, arr, len(others)))

    def seal(self):
        self.sealed = True

    def __len__(self):
        return int(_lib.lib().b200_set_count(self._h))

    @property
    def count(self):
        return len(self)

    nan_count = property(lambda self: int(_lib.lib().b200_set_nan_count(self._h)))
    null_count = property(lambda self: int(_lib.lib().b200_set_null_count(self._h)))
    has_nan = property(lambda self: self.nan_count > 0)
    has_null = property(lambda self: self.null_count > 0)
    nan_index = property(lambda self: int(_lib.lib().b200_set_nan_index(self._h)))
    null_index = property(lambda self: int(_lib.lib().b200_set_null_index(self._h)))

    @property
    def offset(self):
        return int(self.null_count > 0) + int(self.nan_count > 0)  # src/hash.hpp:355-358

    def offsets(self):
        out = np.zeros(self.nmaps, np.int64)
        _lib.check(_lib.lib().b200_set_offsets(self._h, out.ctypes.data))
        return out.tolist()

    def key_array(self):
        out = np.empty(len(self), self._np_dtype())
        if len(out):
            _lib.check(_lib.lib().b200_set_key_array(self._h, out.ctypes.data))
        return out

    def keys(self):
        # hash_common::keys (src/hash.hpp:290-317): python list with nan / None in the special slots
        ar = self.key_array()
        out = ar.tolist()
        if self.nan_count:
            out[self.nan_index] = math.nan
        if self.null_count:
            out[self.null_index] = None
        return out

    def map_ordinal(self, values):
        col = self._key_column(values)
        odt = np.dtype(_lib.DTYPES[_lib.lib().b200_set_ordinal_dtype(self._h)])
        if col.memspace == _lib.MEM_DEVICE:
            import torch
            out = torch.empty(col.length, dtype=getattr(torch, odt.name), device=f"cuda:{self._ctx.device}")
            _lib.check(_lib.lib().b200_set_map_ordinal(self._h, 0, col.ptr, col.length, out.data_ptr(), _lib.MEM_DEVICE, 0))
            self._ctx.sync(0)
            return out
        out = np.empty(col.length, odt)
        if col.length:
            _lib.check(_lib.lib().b200_set_map_ordinal(self._h, 0, col.ptr, col.length, out.ctypes.data, _lib.MEM_HOST, 0))
        return out

    def map_many(self, values, offset, length, output):
        """hash_map<T>::map_many (src/hash_primitives.hpp:567-590), the C++-side interface BinnerHash uses: the GLOBAL ordinals of
        values[offset:offset+length] as int64 into `output` — NaN -> the NaN ordinal (or -1 when the set holds none), absent -> -1;
        masked values are the caller's business."""
        ordinals = self.map_ordinal(values[offset:offset + length])
        if not isinstance(ordinals, np.ndarray):
            ordinals = ordinals.cpu().numpy()
        np.asarray(output)[:length] = ordinals.astype(np.int64)
        return output

    def isin(self, values):
        col = self._key_column(values)
        out = np.empty(col.length, np.uint8)
        if col.memspace == _lib.MEM_DEVICE:
            import torch
            t = torch.empty(col.length, dtype=torch.uint8, device=f"cuda:{self._ctx.device}")
            _lib.check(_lib.lib().b200_set_isin(self._h, 0, col.ptr, col.length, t.data_ptr(), _lib.MEM_DEVICE, 0))
            self._ctx.sync(0)
            return t.bool()
        if col.length:
            _lib.check(_lib.lib().b200_set_isin(self._h, 0, col.ptr, col.length, out.ctypes.data, _lib.MEM_HOST, 0))
        return out.astype(bool)

    def flatten_values(self, values, map_index, out):
        # hash_common::flatten_values (src/hash.hpp:267-288)
        values = np.asarray(values)
        map_index = np.asarray(map_index)
        if values.size != out.size:
            raise RuntimeError("output array does not match length of values")
        if values.size != map_index.size:
            raise RuntimeError("map_index array does not match length of values")
        out[:] = values + np.asarray(self.offsets(), np.int64)[map_index]
        return out

    def extract(self):
        keys = self.key_array()
        offsets = self.offsets() + [len(self)]
        maps = []
        for m in range(self.nmaps):
            d = {}
            for i in range(offsets[m], offsets[m + 1]):
                if (self.nan_count and i == self.nan_index) or (self.null_count and i == self.null_index):
                    continue
                d[keys[i].item()] = i - offsets[m]
            maps.append(d)
        return maps

    def __sizeof__(self):
        return int(_lib.lib().b200_set_bytes(self._h))


def _pickle(x):
    # vaex/hash.py:21-25
    return type(x), (x.key_array(), x.null_index, x.nan_count, x.null_count, x.fingerprint)


for _name in _lib.DTYPES:
    _cls = type("ordered_set_" + _name, (_OrderedSet,), dict(_dtype=_name, _code=_lib.DTYPE_CODE[_name]))
    _cls.__module__ = __name__
    globals()["ordered_set_" + _name] = _cls
    copyreg.pickle(_cls, _pickle)


class _Counter(_OrderedSet):
    """``vaex.superutils.counter_<dtype>`` (src/hash_primitives.hpp:344-433, bound in src/hash_primitives.cpp:36-43): key ->
    number of occurrences — what ``value_counts`` / ``unique`` run on (vaex/cpu.py:141-283).  Layout of ``keys()`` /
    ``key_array()`` / ``counts()``: NaN first, then null, then the keys (the reference lists the keys in its container's
    iteration order, which is unspecified; here they come in first-seen order)."""

    def __init__(self, nmaps=1):
        self._ctx = _lib.context()
        self._h = C.c_void_p()
        self.fingerprint = ""
        self.sealed = False
        self.nmaps = int(nmaps)
        _lib.check(_lib.lib().b200_counter_create(self._ctx._h, self._code, self.nmaps, C.byref(self._h)))

    def _order(self):
        """ordinal positions reordered to the counter layout [nan][null][keys...]"""
        n = len(self)
        special = []
        if self.nan_count:
            special.append(_OrderedSet.nan_index.fget(self))
        if self.null_count:
            special.append(_OrderedSet.null_index.fget(self))
        rest = [i for i in range(n) if i not in special]
        return np.array(special + rest, dtype=np.int64)

    nan_index = property(lambda self: 0)                                  # src/hash.hpp:289
    null_index = property(lambda self: 1 if self.nan_count else 0)        # src/hash.hpp:290

    def key_array(self):
        return _OrderedSet.key_array(self)[self._order()] if len(self) else _OrderedSet.key_array(self)

    def counts(self):
        n = len(self)
        out = np.zeros(n, np.int64)
        if n:
            _lib.check(_lib.lib().b200_set_counts(self._h, out.ctypes.data))
            out = out[self._order()]
        return out

    def keys(self):
        out = self.key_array().tolist()
        if self.nan_count:
            out[0] = math.nan
        if self.null_count:
            out[self.null_index] = None
        return out

    def map_ordinal(self, values):
        raise AttributeError("counter has no map_ordinal")


for _name in _lib.DTYPES:
    _cls = type("counter_" + _name, (_Counter,), dict(_dtype=_name, _code=_lib.DTYPE_CODE[_name]))
    _cls.__module__ = __name__
    globals()["counter_" + _name] = _cls


def device_cast(keys, dtype, ctx):
    """a device key column of another dtype as `dtype`, cast by value where numpy would cast it safely; anything else is a TypeError"""
    import torch
    have = _lib.dtype_of(keys)
    if not np.can_cast(have, dtype, "safe"):
        raise TypeError(f"map_index: incompatible key dtype {have} (index dtype {dtype})")
    ctx.sync()  # a device expression's block is written on a slot's stream
    out = torch.as_tensor(keys, device=f"cuda:{ctx.device}").to(getattr(torch, dtype.name))
    torch.cuda.synchronize(out.device)  # the cast runs on torch's stream, the lookup on a slot's
    return out


_INDEX_OUT = {np.dtype(t): np.dtype(t).itemsize for t in ("int8", "int16", "int32", "int64")}


class _IndexHash:
    """``vaex.superutils.index_hash_<dtype>(nmaps)`` (src/hash_primitives.hpp:731-1040, bound in src/hash_primitives.cpp:57-75):
    key -> row number, what ``df.join`` runs on.  A key's primary row is its smallest row (``start_index + i``) and its other rows
    are its overflow, in ascending order; the NaN / null row is the largest NaN / null row seen.  That is the reference run
    sequentially, one ``update`` per chunk in order, whatever order the chunks arrive in; where the reference's own answer depends
    on chunk order (merges, NaN / null rows of later calls), DESIGN.md states the difference."""
    _dtype = None
    _code = None
    _key_column = _OrderedSet._key_column
    __del__ = _OrderedSet.__del__

    @classmethod
    def _np_dtype(cls):
        return np.dtype(cls._dtype)

    def __init__(self, nmaps=1):
        self._ctx = _lib.context()
        self._h = C.c_void_p()
        self.sealed = False
        self.nmaps = int(nmaps)
        _lib.check(_lib.lib().b200_index_create(self._ctx._h, self._code, self.nmaps, C.byref(self._h)))

    def _lookup_column(self, values):
        """map_index takes ``py::array_t<T>`` without forcecast: numpy converts only where the cast is safe (int32 keys on an int64
        index), anything else is a TypeError.  Device columns follow the same rule: one of another dtype is cast by value on the
        device where numpy calls that safe, and refused otherwise, so a key never reads differently on the host and the device (int8
        -1 is not 255 on a uint8 index, uint64 2^63 not INT64_MIN on an int64 one)."""
        native = self._np_dtype()
        if _lib.is_device(values):
            have = _lib.dtype_of(values)
            if have == native:
                return self._key_column(values)
            return self._key_column(device_cast(values, native, self._ctx))
        if not isinstance(values, np.ndarray):
            values = np.asarray(values, dtype=native)
        if not np.can_cast(values.dtype, native, "safe"):
            raise TypeError(f"{type(self).__name__}.map_index: incompatible key dtype {values.dtype} (index dtype {native})")
        return self._key_column(values)

    def _info(self):
        out = np.zeros(8, np.int64)
        _lib.check(_lib.lib().b200_index_info(self._h, out.ctypes.data))
        return out

    # -- reference protocol --------------------------------------------------------------------------
    def update(self, values, *args, **kwargs):
        """update(values[, masks], start_index=0, chunk_size=..., bucket_size=..., return_values=False); the keyword `slot` (this
        project's addition) names the context slot whose stream the call runs on, so the executor's threads update one index at once"""
        names = ["start_index", "chunk_size", "bucket_size", "return_values"]
        masks = kwargs.pop("masks", None)
        slot = int(kwargs.pop("slot", 0))
        args = list(args)
        if args and not isinstance(args[0], (int, np.integer, bool)):
            masks = args.pop(0)
        opts = dict(start_index=0, chunk_size=1024 * 128, bucket_size=1024 * 128, return_values=False)
        opts.update(zip(names, args))
        opts.update(kwargs)
        if opts["bucket_size"] < opts["chunk_size"]:
            raise RuntimeError("bucket size should be larger than chunk_size")
        if opts["return_values"]:
            raise RuntimeError("index_hash: return_values is not supported")
        if self.sealed:
            raise RuntimeError("hashmap is sealed, cannot update")
        col = self._key_column(values)
        mcol = None
        if masks is not None:
            mcol = _lib.mask_column(masks)
            if mcol.length != col.length:
                raise RuntimeError("array and mask should be of same size")
        _lib.check(_lib.lib().b200_index_update(self._h, slot, col.ptr, None if mcol is None else mcol.ptr, col.length, int(opts["start_index"]),
                                                _lib.memspace(col, mcol), 0))

    def merge(self, other):
        if self.sealed:
            raise RuntimeError("hashmap is sealed, cannot merge")
        others = other if isinstance(other, (list, tuple)) else [other]
        arr = (C.c_void_p * len(others))(*[o._h for o in others])
        _lib.check(_lib.lib().b200_index_merge(self._h, arr, len(others)))

    def _map(self, values, mask, out, slot=0):
        col = self._lookup_column(values)
        mcol = None if mask is None else _lib.mask_column(mask)
        if mcol is not None and mcol.length != col.length:
            raise RuntimeError("array and mask should be of same size")
        give = out is None
        if give:
            if col.memspace == _lib.MEM_DEVICE:
                import torch
                out = torch.empty(col.length, dtype=torch.int64, device=f"cuda:{self._ctx.device}")
            else:
                out = np.empty(col.length, np.int64)
        ocol = _lib.column(out)
        if ocol.dtype not in _INDEX_OUT or ocol.length < col.length:
            raise TypeError(f"map_index: out must be an int8, int16, int32 or int64 array of at least {col.length} rows")
        unknown = C.c_int32(0)
        if col.length:
            _lib.check(_lib.lib().b200_index_map(self._h, slot, col.ptr, None if mcol is None else mcol.ptr, col.length, ocol.ptr, _INDEX_OUT[ocol.dtype],
                                                 C.byref(unknown), _lib.memspace(col, mcol, ocol), 0))
        if isinstance(out, np.ndarray) and ocol.keep is not out:
            out[:] = ocol.keep  # a non-contiguous host `out` was written through a copy
        return out if give else bool(unknown.value)

    def map_index(self, values, out=None, slot=0):
        """map_index(values) -> int64 rows (-1: not found); map_index(values, out) writes int8..int64 ``out`` (truncating) and returns
        whether a key was not found"""
        return self._map(values, None, out, slot)

    def map_index_masked(self, values, mask, out=None, slot=0):
        return self._map(values, mask, out, slot)

    def map_index_duplicates(self, values, start_index, mask=None, device=False, slot=0):
        """(left rows, right rows): for every row i of `values` whose key has an overflow, ``start_index + i`` paired with each overflow
        row.  `mask` (masked rows contribute none) and `device` (torch results on the index's GPU) are this project's additions."""
        col = self._lookup_column(values)
        mcol = None if mask is None else _lib.mask_column(mask)
        lib, ms = _lib.lib(), _lib.memspace(col, mcol)
        total = C.c_int64(0)
        args = (self._h, slot, col.ptr, None if mcol is None else mcol.ptr, col.length, int(start_index))
        _lib.check(lib.b200_index_duplicates(*args, None, None, 0, C.byref(total), ms, 0))
        while True:  # the pairs are written only when they fit: an update from another thread in between changes the total
            n = total.value
            if device:
                import torch
                left, right = (torch.empty(n, dtype=torch.int64, device=f"cuda:{self._ctx.device}") for _ in range(2))
                lp, rp = left.data_ptr(), right.data_ptr()
            else:
                left, right = np.empty(n, np.int64), np.empty(n, np.int64)
                lp, rp = left.ctypes.data, right.ctypes.data
            if not n:
                break
            _lib.check(lib.b200_index_duplicates(*args, lp, rp, n, C.byref(total), _lib.memspace(col, mcol, _lib.column(left)), 0))
            if total.value == n:
                break
        return left, right

    has_duplicates = property(lambda self: bool(self._info()[2]))
    nan_count = property(lambda self: int(self._info()[3]))
    null_count = property(lambda self: int(self._info()[4]))
    has_nan = property(lambda self: self.nan_count > 0)
    has_null = property(lambda self: self.null_count > 0)
    count = property(lambda self: int(self._info()[1]))

    def __len__(self):
        return int(self._info()[0])

    def _nan_row(self):
        return int(self._info()[5])

    def _null_row(self):
        return int(self._info()[6])

    def seal(self):
        self.sealed = True

    def _extract_arrays(self):
        n = C.c_int64(0)
        _lib.check(_lib.lib().b200_index_extract(self._h, None, None, None, 0, C.byref(n)))
        while True:  # written only when it fits: an update from another thread in between changes the count
            cap = n.value
            keys, rows, shards = np.empty(cap, np.uint64), np.empty(cap, np.int64), np.empty(cap, np.int16)
            _lib.check(_lib.lib().b200_index_extract(self._h, keys.ctypes.data, rows.ctypes.data, shards.ctypes.data, cap, C.byref(n)))
            if n.value <= cap:
                keys, rows, shards = keys[:n.value], rows[:n.value], shards[:n.value]
                break
        native = self._np_dtype()
        keys = keys.astype(np.dtype(f"u{native.itemsize}")).view(native)  # canonical patterns -> the key's own bits
        return keys, rows, shards

    def extract(self):
        keys, rows, shards = self._extract_arrays()
        maps = [{} for _ in range(self.nmaps)]
        for k, r, m in zip(keys.tolist(), rows.tolist(), shards.tolist()):
            maps[m][k] = r
        return maps

    def offsets(self):
        # hash_common::offsets (src/hash.hpp:337-353): shard 0 also holds the NaN / null entries
        _, _, shards = self._extract_arrays()
        sizes = np.bincount(shards, minlength=self.nmaps).astype(np.int64)
        sizes[0] += self.offset
        return [0] + np.cumsum(sizes)[:-1].tolist()

    @property
    def offset(self):
        return int(self.null_count > 0) + int(self.nan_count > 0)

    def __sizeof__(self):
        return int(self._info()[7])


for _name in _lib.DTYPES:
    _cls = type("index_hash_" + _name, (_IndexHash,), dict(_dtype=_name, _code=_lib.DTYPE_CODE[_name]))
    _cls.__module__ = __name__
    globals()["index_hash_" + _name] = _cls


# ---- string keys (src/hash_string.hpp, bound in src/hash_string.cpp:86-99 as ordered_set_string) ------------------------------------
def string_buffers(values):
    """strings -> (int64 offsets[n + 1], uint8 bytes, uint8 null mask or None): the arrow large_string layout the reference's
    StringList64 uses.  Accepts pyarrow string / large_string arrays (zero copy for large_string), numpy object / str arrays and
    lists of str / None."""
    try:
        import pyarrow as pa
    except ImportError:  # pragma: no cover
        pa = None
    if pa is not None and isinstance(values, pa.ChunkedArray):
        values = values.combine_chunks()
    if pa is not None and isinstance(values, pa.Array):
        if pa.types.is_string(values.type):
            values = values.cast(pa.large_string())
        if not pa.types.is_large_string(values.type):
            raise TypeError(f"expected a string array, got {values.type}")
        n = len(values)
        validity, off_buf, data_buf = values.buffers()
        offsets = np.frombuffer(off_buf, dtype=np.int64, count=n + 1, offset=values.offset * 8)
        data = np.frombuffer(data_buf, dtype=np.uint8) if data_buf is not None else np.zeros(0, np.uint8)
        mask = None
        if values.null_count:
            bits = np.unpackbits(np.frombuffer(validity, dtype=np.uint8), bitorder="little")[values.offset:values.offset + n]
            mask = np.ascontiguousarray(1 - bits).astype(np.uint8)
        return offsets, data, mask
    seq = values.tolist() if isinstance(values, np.ndarray) else list(values)
    enc = [(s.encode("utf8") if s is not None else b"") for s in seq]
    offsets = np.zeros(len(enc) + 1, np.int64)
    if enc:
        offsets[1:] = np.cumsum([len(e) for e in enc])
    data = np.frombuffer(b"".join(enc), dtype=np.uint8).copy() if offsets[-1] else np.zeros(0, np.uint8)
    mask = np.array([s is None for s in seq], np.uint8)
    return offsets, data, (mask if mask.any() else None)


class ordered_set_string:
    """``vaex.superutils.ordered_set_string(nmaps, limit=-1)``: the ordinal encoder for string keys, on the device.
    update / map_ordinal / key_array / keys / offsets / len / null_count / has_null / null_index follow the reference
    (src/hash_string.hpp); ``limit``, ``isin``, ``merge`` and ``flatten_values`` are not provided."""

    def __init__(self, nmaps=1, limit=-1):
        self._ctx = _lib.context()
        self._h = C.c_void_p()
        self.nmaps = int(nmaps)
        self.fingerprint = ""
        self.sealed = False
        _lib.check(_lib.lib().b200_strset_create(self._ctx._h, self.nmaps, int(limit), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().b200_set_destroy(h)
            except Exception:
                pass
            self._h = None

    @staticmethod
    def _np_dtype():
        return np.dtype("O")

    def update(self, values, start_index=0, chunk_size=1024 * 128, bucket_size=1024 * 128, return_values=False, slot=0):
        if self.sealed:
            raise RuntimeError("cannot add to sealed hashmap")
        if bucket_size < chunk_size:
            raise RuntimeError("bucket size should be larger than chunk_size")
        offsets, data, mask = string_buffers(values)
        n = len(offsets) - 1
        vals = np.empty(n if return_values else 1, np.int64)
        mi = np.empty(n if return_values else 1, np.int16)
        _lib.check(_lib.lib().b200_strset_update(self._h, self._ctx.slot(slot), offsets.ctypes.data, data.ctypes.data if data.size else None,
                                                 None if mask is None else mask.ctypes.data, n, int(bool(return_values)), vals.ctypes.data, mi.ctypes.data, _lib.MEM_HOST))
        return (vals, mi) if return_values else None

    def map_ordinal(self, values, slot=0, device=False):
        """global ordinals, -1 for strings that are not members; device=True returns a device array (for the fused groupby pass)"""
        offsets, data, mask = string_buffers(values)
        n = len(offsets) - 1
        args = (offsets.ctypes.data, data.ctypes.data if data.size else None, None if mask is None else mask.ctypes.data, n)
        if device:
            import torch
            from .expression import DeviceArray
            buf = torch.empty(max(n, 1), dtype=torch.int64, device=f"cuda:{self._ctx.device}")
            _lib.check(_lib.lib().b200_strset_map_ordinal(self._h, self._ctx.slot(slot), *args, buf.data_ptr(), _lib.MEM_HOST, 1))
            return DeviceArray(buf.data_ptr(), n, np.int64, keep=buf)
        out = np.empty(n, np.int64)
        _lib.check(_lib.lib().b200_strset_map_ordinal(self._h, self._ctx.slot(slot), *args, out.ctypes.data, _lib.MEM_HOST, 0))
        return out

    def _key_buffers(self):
        n = len(self)
        nbytes = C.c_int64(0)
        _lib.check(_lib.lib().b200_strset_key_bytes(self._h, C.byref(nbytes)))
        offsets = np.zeros(n + 1, np.int64)
        data = np.zeros(max(nbytes.value, 1), np.uint8)
        _lib.check(_lib.lib().b200_strset_key_array(self._h, offsets.ctypes.data, data.ctypes.data))
        return offsets, data[:nbytes.value]

    def key_array(self):
        """the keys in ordinal order as a pyarrow large_string array (the reference hands out a StringList64); the null slot is null"""
        import pyarrow as pa
        offsets, data = self._key_buffers()
        n = len(offsets) - 1
        validity = None
        if self.null_count:
            bits = np.ones(n, np.uint8)
            bits[self.null_index] = 0
            validity = pa.py_buffer(np.packbits(bits, bitorder="little").tobytes())
        return pa.Array.from_buffers(pa.large_string(), n, [validity, pa.py_buffer(offsets.tobytes()), pa.py_buffer(data.tobytes())], null_count=1 if self.null_count else 0)

    def keys(self):
        return self.key_array().to_pylist()

    def seal(self):
        self.sealed = True

    def __len__(self):
        return int(_lib.lib().b200_set_count(self._h))

    count = property(lambda self: len(self))
    nan_count = property(lambda self: 0)
    null_count = property(lambda self: int(_lib.lib().b200_set_null_count(self._h)))
    has_nan = property(lambda self: False)
    has_null = property(lambda self: self.null_count > 0)
    nan_index = property(lambda self: -1)
    null_index = property(lambda self: int(_lib.lib().b200_set_null_index(self._h)))  # 0x7fffffff until a null was seen

    @property
    def offset(self):
        return int(self.null_count > 0)

    def offsets(self):
        out = np.zeros(self.nmaps, np.int64)
        _lib.check(_lib.lib().b200_set_offsets(self._h, out.ctypes.data))
        return out.tolist()


def create_set_string(keys, null_index=-1, nan_count=0, null_count=0, fingerprint=""):
    """vaex/hash.py:28-36: an ordered_set_string rebuilt from its keys in ordinal order (a pyarrow string array whose null slot, if
    any, is the null key) — one shard, so ordinal == position again."""
    s = ordered_set_string(1)
    # a null takes the ordinal at the END of the update call that first sees it (src/hash_string.hpp): feed the keys up to and
    # including the null slot in one call, the rest in a second one, and every key is back at its position
    if null_count and 0 <= null_index < len(keys) - 1:
        s.update(keys[:null_index + 1])
        s.update(keys[null_index + 1:])
    elif len(keys):
        s.update(keys)
    s.fingerprint = fingerprint
    return s


def _pickle_set_string(x):
    return create_set_string, (x.key_array(), x.null_index, 0, x.null_count, x.fingerprint)


copyreg.pickle(ordered_set_string, _pickle_set_string)
