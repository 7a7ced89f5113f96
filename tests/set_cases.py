"""Edge corpus for the ordered sets / counters (vaex_b200.superutils.ordered_set_<T>, counter_<T>).

Per dtype: key columns that mix the values where a hashed key path goes wrong -- the key whose canonical 64-bit pattern is the
device table's empty marker (uint64 2^64-1, or -1 of a signed type after sign extension), the limits of the type, uint64 >= 2^63,
+-0.0, +-inf, subnormals, the largest finite values and NaNs of every payload (negative, signalling, all-ones) -- with masks, long
runs of one key, all-distinct keys and keys whose first occurrence comes late in a call.  `sequences()` turns them into update
calls (several calls, start_index -1 / 0, return_values).

Used by tests/test_set_edges_cpu.py (oracle against the compiled reference), tests/golden/make_golden_set_edges.py (known answers
of the compiled reference) and tests/test_gpu_hash_edges.py (the device against both)."""
import numpy as np

DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"]
NMAPS = [1, 2, 3, 7, 255, 256, 257, 1000, 32767]

F64_NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0x7FF4000000000000]
F32_NAN_BITS = [0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0xFFFFFFFF, 0x7FA00000]


def sentinel(dtype):
    """the key whose canonical pattern is 2^64-1 (None for types that cannot produce it)"""
    dt = np.dtype(dtype)
    if dt.kind == "i":
        return dt.type(-1)
    if dt == np.uint64:
        return np.uint64(2 ** 64 - 1)
    return None


def nan_values(dtype):
    dt = np.dtype(dtype)
    if dt == np.float64:
        return np.array(F64_NAN_BITS, np.uint64).view(np.float64)
    if dt == np.float32:
        return np.array(F32_NAN_BITS, np.uint32).view(np.float32)
    return np.zeros(0, dt)


def edge_values(dtype, zeros=True):
    """the finite / infinite / integer edge values of a dtype (no NaN).  zeros=False leaves out -0.0: the compiled reference
    merges +0.0 and -0.0 in small tables only (a documented deviation), so bit-for-bit comparisons with it skip -0.0."""
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return np.array([False, True])
    if dt.kind == "f":
        fi = np.finfo(dt)
        v = [0.0, 1.0, -1.0, np.inf, -np.inf, fi.max, -fi.max, fi.tiny, -fi.tiny, fi.smallest_subnormal, -fi.smallest_subnormal,
             fi.smallest_subnormal * 3, fi.eps, 0.5, 2.0 ** 20 + 0.5]
        if zeros:
            v.append(-0.0)
        return np.array(v, dt)
    ii = np.iinfo(dt)
    v = {0, 1, 2, ii.max, ii.max - 1, ii.min, ii.min + 1, 127, 128, 255, 256, 32767, 32768, 65535}
    if dt.kind == "i":
        v |= {-1, -2, -128, -129}
    if dt == np.uint64:
        v |= {2 ** 63, 2 ** 63 - 1, 2 ** 63 + 1, 2 ** 64 - 2}
    return np.array(sorted(x for x in v if ii.min <= x <= ii.max), dtype=dt)


def _filler(rng, dtype, n, lo=-300, hi=300):
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return rng.integers(0, 2, n).astype(dt)
    if dt.kind == "f":
        return (rng.integers(lo, hi, n) * 0.25).astype(dt)
    ii = np.iinfo(dt)
    return rng.integers(max(ii.min, lo), min(ii.max, hi) + 1, n).astype(dt)


def columns(dtype, seed=0, zeros=True, n=3000):
    """[(name, keys, mask or None)]: the edge-corpus key columns of one dtype"""
    dt = np.dtype(dtype)
    rng = np.random.default_rng([seed, DTYPES.index(dt.name)])
    edges = edge_values(dt, zeros)
    nans = nan_values(dt)
    special = np.concatenate([edges, nans]) if len(nans) else edges
    out = []
    # every edge value (and NaN payload) several times, shuffled into filler, with masked rows
    k = np.concatenate([np.repeat(special, 3), _filler(rng, dt, n)])
    rng.shuffle(k)
    out.append(("mixed", k, rng.random(len(k)) < 0.04))
    # a long run of the sentinel (or the first edge value), then the rest once
    head = sentinel(dt) if sentinel(dt) is not None else edges[-1]
    out.append(("run", np.concatenate([np.full(n, head, dt), special]), None))
    # all distinct: edges first, then a range of values not among them
    if dt.kind == "b":
        distinct = edges
    elif dt.kind == "f":
        distinct = np.concatenate([edges, (np.arange(n) + 0.125).astype(dt) * 3])
    else:
        ii = np.iinfo(dt)
        span = np.arange(min(n, ii.max // 2), dtype=np.int64) * 2 + 3
        distinct = np.unique(np.concatenate([edges, span.astype(dt)]))
        rng.shuffle(distinct)
    out.append(("distinct", distinct, None))
    # first occurrences late: a few filler keys repeated, the edge values (and NaN) only in the last rows, a masked row in between
    late = np.concatenate([np.repeat(_filler(rng, dt, 7, 3, 9), n // 7), special[::-1]])
    m = np.zeros(len(late), bool)
    m[len(late) - len(special) - 1] = True
    out.append(("late", late, m))
    return out


def sequences(dtype, seed=0, zeros=True, n=3000):
    """[(name, [call, ...])]: update sequences; a call is dict(keys, mask, start_index, return_values)"""
    cols = columns(dtype, seed, zeros, n)
    rng = np.random.default_rng([seed, 99, DTYPES.index(np.dtype(dtype).name)])
    seqs = []
    for name, k, m in cols:
        seqs.append((name, [dict(keys=k, mask=m, start_index=0, return_values=True)]))
    # several calls over all columns: alternate start_index (NaN / null order), one with return_values
    calls = []
    for i, (name, k, m) in enumerate(cols):
        calls.append(dict(keys=k, mask=m, start_index=int(rng.choice([-1, 0])), return_values=i == 2))
    seqs.append(("calls", calls))
    # NaN / null first seen in a later call, after the sentinel
    s = sentinel(dtype)
    first = np.array([s if s is not None else edge_values(dtype)[0]] * 5, np.dtype(dtype))
    nans = nan_values(dtype)
    second = np.concatenate([edge_values(dtype, zeros), nans[:2]]) if len(nans) else edge_values(dtype, zeros)
    m2 = np.zeros(len(second), bool)
    m2[1] = True
    seqs.append(("specials_later", [dict(keys=first, mask=None, start_index=-1, return_values=False),
                                     dict(keys=second, mask=m2, start_index=-1, return_values=False),
                                     dict(keys=second[::-1].copy(), mask=None, start_index=0, return_values=True)]))
    return seqs


def queries(dtype, zeros=True):
    """keys to look up after an update: every edge value and NaN payload plus values that are never inserted"""
    dt = np.dtype(dtype)
    q = [edge_values(dt, zeros), nan_values(dt)]
    if dt.kind == "f":
        q.append(np.array([7.75e3, -7.75e3, 1e-30], dt))
    elif dt.kind in "iu":
        ii = np.iinfo(dt)
        q.append(np.array([min(ii.max, 99991), ii.max - 3, max(ii.min, 4)], dt))
    return np.concatenate(q)


# ---- strings built to hit the string set's refusal paths --------------------------------------------------------------------
# libstdc++'s 64-bit _Hash_bytes (the reference's std::hash<string_view>) on whole 8-byte blocks can be undone step by step: the
# multiplies are by an odd constant (invertible mod 2^64) and x ^= x >> 47 is its own inverse.
_MUL = ((0xC6A4A793 << 32) + 0x5BD1E995)
_MASK = (1 << 64) - 1
_INV = pow(_MUL, -1, 1 << 64)
_SEED = 0xC70F6907


def _unshift47(x):
    return x ^ (x >> 47)


def _mix(block):
    d = (block * _MUL) & _MASK
    d ^= d >> 47
    return (d * _MUL) & _MASK


def _unmix(d):
    d = (d * _INV) & _MASK
    d = _unshift47(d)
    return (d * _INV) & _MASK


def _state_after(prefix, n):
    """the hash state after the whole 8-byte blocks of `prefix`, for a string of total length n"""
    h = (_SEED ^ ((n * _MUL) & _MASK)) & _MASK
    for p in range(0, len(prefix), 8):
        h = ((h ^ _mix(int.from_bytes(prefix[p:p + 8], "little"))) * _MUL) & _MASK
    return h


def last_block_for(prefix, target):
    """the 8 bytes b such that hash(prefix + b) == target (len(prefix) a multiple of 8)"""
    n = len(prefix) + 8
    h = _unshift47(target)
    h = (h * _INV) & _MASK
    h = _unshift47(h)
    h = (h * _INV) & _MASK  # == state_before_last ^ mix(block)
    return _unmix(h ^ _state_after(prefix, n)).to_bytes(8, "little")


def ascii_string_with_hash(target, tag=b"", tries=1 << 16):
    """a 16-byte ASCII string whose std::hash is `target`: the first block is free, the second one solved; tried until that one is
    ASCII as well (one try in 256 on average)"""
    for i in range(tries):
        first = (tag + b"%07d" % i)[-8:].rjust(8, b"_")
        last = last_block_for(first, target)
        if all(32 <= c < 127 for c in last):
            return (first + last).decode("ascii")
    raise RuntimeError("no ASCII preimage found")


def ascii_collision(other, tries=1 << 16):
    """a 16-byte ASCII string other than `other` (16 ASCII bytes) with the same std::hash"""
    from oracle.oracle import string_hash
    target = string_hash(other.encode("ascii"))
    s = ascii_string_with_hash(target, b"c", tries)
    assert s != other
    return s


# ---- the numpy restatement used for big cases ------------------------------------------------------------------------------
_M1, _M2 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def hash64(x):
    """splitmix64 finaliser (the reference's _hash64, src/hash.hpp:40-45) on a uint64 array"""
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = (x ^ (x >> np.uint64(30))) * _M1
        x = (x ^ (x >> np.uint64(27))) * _M2
    return x ^ (x >> np.uint64(31))


def canon(keys):
    """key -> canonical 64-bit pattern (signed types sign-extended, the rest zero-extended)"""
    k = np.asarray(keys)
    if k.dtype.kind == "i":
        return k.astype(np.int64).view(np.uint64)
    if k.dtype.kind == "f":
        return k.view(np.uint64 if k.dtype.itemsize == 8 else np.uint32).astype(np.uint64)
    return k.astype(np.uint64)


def shard_of(keys, nmaps):
    k = np.asarray(keys)
    c = canon(k)
    h = c if (k.dtype.itemsize <= 2) else hash64(c)
    return (h % np.uint64(nmaps)).astype(np.int64)


def restate(calls, dtype, nmaps):
    """ordered_set state after `calls` (lists of (keys, mask)) for keys WITHOUT NaN: per shard key % nmaps the ordinal is the rank
    of first occurrence; a null goes to shard 0 at the end of the call that first saw one (the NaN does the same, which needs no
    case here).  Returns (key_array, offsets, null_index or None, null_count)."""
    dt = np.dtype(dtype)
    parts, seen = [], set()
    null_count, null_call = 0, None
    for ci, (k, m) in enumerate(calls):
        k = np.asarray(k, dt)
        valid = k if m is None else k[~m]
        parts.append(valid)
        if m is not None and m.any():
            null_count += int(m.sum())
            if null_call is None:
                null_call = ci
    allk = np.concatenate(parts) if parts else np.zeros(0, dt)
    call_of = np.concatenate([np.full(len(p), i) for i, p in enumerate(parts)]) if parts else np.zeros(0, np.int64)
    u, first = np.unique(allk, return_index=True)
    order = np.argsort(first, kind="stable")
    keys, first, calls_first = u[order], first[order], call_of[first[order]]
    shard = shard_of(keys, nmaps)
    # the null sorts into shard 0 behind every key of the call that first saw it
    null_pos = None
    if null_call is not None:
        in0 = np.flatnonzero((shard == 0) & (calls_first <= null_call))
        null_pos = len(in0)
    so = np.argsort(shard, kind="stable")
    keys, shard = keys[so], shard[so]
    counts = np.bincount(shard, minlength=nmaps)
    if null_pos is not None:
        keys = np.insert(keys, null_pos, np.array([-1]).astype(dt))  # the null slot holds (T)-1
        counts[0] += 1
    offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).tolist()
    return keys, offsets, null_pos, null_count
