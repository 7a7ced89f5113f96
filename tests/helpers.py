"""Shared helpers: run the same spec dicts (oracle.scalar/ordinal/agg) through the product (vaex_b200.superagg)."""
import numpy as np


def _suffix(ar):
    ar = np.asarray(ar) if not hasattr(ar, "__cuda_array_interface__") or isinstance(ar, np.ndarray) else ar
    dt = np.dtype(ar.dtype) if isinstance(ar, np.ndarray) else np.dtype(str(ar.dtype).replace("torch.", ""))
    name = dt.newbyteorder("=").name
    swapped = dt.byteorder not in ("=", "|") and dt.byteorder != ("<" if np.little_endian else ">")
    return name + ("_non_native" if swapped else "")


def to_device(ar):
    """numpy -> torch CUDA tensor (byte-swapped arrays are shipped as their raw native-typed bytes)."""
    import torch
    if ar is None:
        return None
    ar = np.ascontiguousarray(ar)
    if ar.dtype == np.bool_:
        return torch.from_numpy(ar).cuda()
    if ar.dtype.kind == "u" and ar.dtype.itemsize > 1:
        # torch has limited unsigned support: move the bytes as the signed type of equal width
        return torch.from_numpy(ar.view(ar.dtype.newbyteorder("=").str.replace("u", "i"))).cuda()
    return torch.from_numpy(ar.view(ar.dtype.newbyteorder("="))).cuda()


class B200Binby:
    """The product-side twin of oracle.ref_driver.RefBinby: same class names, same call protocol."""

    def __init__(self, binners, aggs, nthreads=1):
        from vaex_b200 import superagg
        self.binner_specs, self.agg_specs, self.nthreads = binners, aggs, nthreads
        self.binners = []
        for b in binners:
            sfx = _suffix(b["data"])
            if b["kind"] == "scalar":
                self.binners.append(getattr(superagg, "BinnerScalar_" + sfx)(nthreads, "x", b["vmin"], b["vmax"], b["bins"]))
            elif b["kind"] == "ordinal":
                self.binners.append(getattr(superagg, "BinnerOrdinal_" + sfx)(nthreads, "x", b["count"], b["min_value"], b["allow_other"], b["invert"]))
            else:
                self.binners.append(getattr(superagg, "BinnerHash_" + sfx)(nthreads, "x", b["set"], b.get("allow_other", False), b.get("invert", False)))
        self.grid = superagg.Grid(self.binners)
        self.aggs = []
        for a in aggs:
            op, data = a["op"], a["data"]
            sfx = "int64" if data is None else _suffix(data)
            if op == "count":
                agg = getattr(superagg, "AggCount_" + sfx)(self.grid, 1, nthreads)
            elif op == "sum":
                agg = getattr(superagg, "AggSum_" + sfx)(self.grid, 1, nthreads)
            elif op == "sum_moment":
                agg = getattr(superagg, "AggSumMoment_" + sfx)(self.grid, 1, nthreads, a["moment"])
            elif op == "min":
                agg = getattr(superagg, "AggMin_" + sfx)(self.grid, 1, nthreads)
            elif op == "max":
                agg = getattr(superagg, "AggMax_" + sfx)(self.grid, 1, nthreads)
            elif op in ("first", "last"):
                order = a.get("order")
                sfx2 = "int64" if order is None else np.asarray(order).dtype.newbyteorder("=").name
                name = "AggFirst_" + np.asarray(data).dtype.newbyteorder("=").name + "_" + sfx2 + ("_non_native" if sfx.endswith("_non_native") else "")
                agg = getattr(superagg, name)(self.grid, 1, nthreads, op == "last")
            elif op == "nunique":
                agg = getattr(superagg, "AggNUnique_" + sfx)(self.grid, 1, nthreads, a.get("dropmissing", False), a.get("dropnan", False))
            else:
                raise ValueError(op)
            self.aggs.append(agg)

    def process(self, thread, i1, i2, device=False):
        """device: False = host numpy chunks; True = each chunk copied to the device; "resident" = every column copied to the
        device once and fed as slices of it (a slice that starts at an odd row is off the 16-byte boundary)"""
        if device == "resident":
            cache = self.__dict__.setdefault("_resident", {})

            def col(x):
                x = np.asarray(x)
                if id(x) not in cache:
                    cache[id(x)] = (x, to_device(x))
                return cache[id(x)][1][i1:i2]
        else:
            conv = to_device if device else (lambda x: x)

            def col(x):
                return conv(np.asarray(x)[i1:i2])
        for binner, spec in zip(self.binners, self.binner_specs):
            binner.set_data(thread, col(spec["data"]))
            if spec.get("mask") is not None:
                binner.set_data_mask(thread, col(spec["mask"]))
            else:
                binner.clear_data_mask(thread)
        for agg, spec in zip(self.aggs, self.agg_specs):
            if spec["data"] is not None:
                agg.set_data(thread, col(spec["data"]), 0)
            if spec.get("order") is not None:
                agg.set_data(thread, col(spec["order"]), 1)
            if spec["mask"] is not None:
                agg.set_data_mask(thread, col(spec["mask"]))
            else:
                agg.clear_data_mask(thread)
            if spec["op"] == "nunique":
                if spec.get("selection") is not None:
                    agg.set_selection_mask(thread, col(spec["selection"]))
                else:
                    agg.clear_selection_mask(thread)
        self.grid.bin(thread, self.aggs, i2 - i1, row_offset=i1)

    def run(self, length, chunk=None, device=False, start=0):
        chunk = chunk or max(length, 1)
        t = 0
        for i1 in range(start, length, chunk):
            self.process(t % self.nthreads, i1, min(i1 + chunk, length), device)
            t += 1
        return [a.get_result() for a in self.aggs]


def b200_binby(binners, aggs, length=None, chunk=None, device=False, nthreads=1):
    if length is None:
        length = len(binners[0]["data"])
    return B200Binby(binners, aggs, nthreads).run(length, chunk, device)


def same(a, b, rtol=0.0):
    """bit-exact for integers / min / max / counts; rtol for floating sums."""
    if np.ma.isMaskedArray(a) or np.ma.isMaskedArray(b):
        ma, mb = np.ma.getmaskarray(a), np.ma.getmaskarray(b)
        return np.array_equal(ma, mb) and same(np.asarray(a.data)[~ma], np.asarray(b.data)[~mb], rtol)
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if rtol and a.dtype.kind == "f":
        return np.allclose(a, b, rtol=rtol, atol=0, equal_nan=True)
    return np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def same_bits(a, b):
    """bit-exact on the raw storage (so -0.0 != +0.0), except that any two NaNs are equal; masked arrays: same mask, same bits
    where unmasked."""
    if np.ma.isMaskedArray(a) or np.ma.isMaskedArray(b):
        ma, mb = np.ma.getmaskarray(a), np.ma.getmaskarray(b)
        return np.array_equal(ma, mb) and same_bits(np.asarray(a.data)[~ma], np.asarray(b.data)[~mb])
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind == "f":
        nan_a, nan_b = np.isnan(a), np.isnan(b)
        if not np.array_equal(nan_a, nan_b):
            return False
        a, b = a[~nan_a], b[~nan_b]
    if a.dtype.kind == "b" or a.dtype.itemsize == 1:
        return np.array_equal(a.view(np.uint8), b.view(np.uint8))
    u = np.dtype("u%d" % a.dtype.itemsize)
    return np.array_equal(np.ascontiguousarray(a).view(u), np.ascontiguousarray(b).view(u))


F64_EDGES = np.array([0.0, -0.0, np.inf, -np.inf, 5e-324, -5e-324, 2.225073858507201e-308, 2.2250738585072014e-308, -2.2250738585072014e-308,
                      1.7976931348623157e308, -1.7976931348623157e308, 1e155, -1e155, 1e80, -1e80, 3e6, 1.0, -1.0])
F64_NANS = np.array([0x7FF8000000000001, 0x7FF0000000000001, 0xFFF8000000000123, 0x7FFFFFFFFFFFFFFF], np.uint64).view(np.float64)
F32_EDGES = np.array([0.0, -0.0, np.inf, -np.inf, 1e-45, -1e-45, 1.1754942e-38, 1.1754944e-38, -1.1754944e-38, 3.4028235e38, -3.4028235e38,
                      1e30, -1e30, 1.0, -1.0], np.float32)
F32_NANS = np.array([0x7FC00001, 0x7F800001, 0xFFC00123, 0x7FFFFFFF], np.uint32).view(np.float32)


def edge_values(dt):
    """the values where kernels go wrong, for one dtype (native byte order)"""
    d = np.dtype(dt).newbyteorder("=")
    if d.kind == "f":
        return np.concatenate([F64_EDGES, F64_NANS]) if d.itemsize == 8 else np.concatenate([F32_EDGES, F32_NANS])
    if d.kind == "b":
        return np.array([False, True])
    info = np.iinfo(d)
    vals = [info.min, info.min + 1, -1, 0, 1, info.max - 1, info.max]
    if d == np.uint64:
        vals += [1 << 63, (1 << 63) + 1, (1 << 64) - 12345, 3_000_000]
    return np.array([v for v in vals if info.min <= v <= info.max], dtype=object).astype(d)


def _mix_edges(rng, data, extra=()):
    """replace about a third of the rows by edge values of the column's dtype (plus `extra`), keep the byte order"""
    n = len(data)
    if not n:
        return data
    d = data.dtype
    pool = edge_values(d)
    if len(extra):
        pool = np.concatenate([pool, np.asarray(extra).astype(pool.dtype)])
    out = data.astype(d.newbyteorder("="))
    at = rng.random(n) < 0.35
    out[at] = pool[rng.integers(0, len(pool), int(at.sum()))]
    return out.astype(d)


def _swapped_twin(rng, data):
    """edge mode: sometimes ship the same values as the byte-swapped twin dtype"""
    if data.dtype.itemsize > 1 and rng.random() < 0.3:
        return data.astype(data.dtype.newbyteorder("S"))
    return data


def random_case(rng, n, allow_first=True, float_sum_ok=True, edges=False):
    """One random (binners, aggs) problem covering every dtype, masks, NaNs, byte order, all aggregators.

    edges=True mixes the values where kernels go wrong into every column (integer limits, uint64 >= 2^63, +-0.0, +-inf, NaN
    payloads, subnormals, the largest finite values, values whose square or 4th power overflows, keys on / next to bin edges),
    sometimes as byte-swapped twins, draws moments 0..8 and adds nunique.  The extra draws only happen in edge mode, so the
    default mode produces the very same cases for a seed as before."""
    from oracle import oracle as O
    nd = int(rng.integers(1, 4))
    binners = []
    for d in range(nd):
        if rng.random() < 0.6:
            dt = rng.choice(["f8", "f4", "i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?", ">f8", ">f4", ">i4", ">u2"])
            if np.dtype(dt).kind == "f":
                data = rng.normal(0, 1, n).astype(dt)
                data[rng.random(n) < 0.01] = np.nan
            elif dt == "?":
                data = rng.integers(0, 2, n).astype(dt)
            else:
                data = rng.integers(-5 if np.dtype(dt).kind == "i" else 0, 20, n).astype(dt)
            mask = (rng.random(n) < 0.1) if rng.random() < 0.5 else None
            bins = int(rng.integers(1, 12))
            if edges:
                e = -2.5 + (3.1 - -2.5) * np.arange(bins + 1) / bins
                data = _swapped_twin(rng, _mix_edges(rng, data, np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf)])
                                                     if np.dtype(dt).kind == "f" else ()))
            binners.append(O.scalar(data, -2.5, 3.1, bins, mask=mask))
        else:
            dt = rng.choice(["i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?", "f8", "f4", ">i4", ">i8"])
            if np.dtype(dt).kind == "f":
                data = rng.integers(-3, 12, n).astype(dt)
                data[rng.random(n) < 0.02] = np.nan
            elif dt == "?":
                data = rng.integers(0, 2, n).astype(dt)
            else:
                data = rng.integers(-3 if np.dtype(dt).kind == "i" else 0, 12, n).astype(dt)
            mask = (rng.random(n) < 0.1) if rng.random() < 0.5 else None
            count, min_value = int(rng.integers(1, 9)), int(rng.integers(-2, 3))
            if edges:
                data = _swapped_twin(rng, _mix_edges(rng, data, [min_value - 1, min_value, min_value + count - 1, min_value + count]
                                                     if np.dtype(dt).kind == "f" else ()))
            binners.append(O.ordinal(data, count, min_value, bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), mask=mask))
    aggs = []
    ops = ["count", "count*", "sum", "sum_moment", "min", "max"] + (["first", "last"] if allow_first else []) + (["nunique"] if edges else [])
    for k in range(int(rng.integers(1, 5))):
        op = rng.choice(ops)
        dt = rng.choice(["f8", "f4", "i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?", ">f8", ">i4"])
        if np.dtype(dt).kind == "f":
            data = rng.normal(0, 10, n).astype(dt)
            data[rng.random(n) < 0.02] = np.nan
        elif dt == "?":
            data = rng.integers(0, 2, n).astype(dt)
        else:
            data = rng.integers(-50 if np.dtype(dt).kind == "i" else 0, 100, n).astype(dt)
        mask = (rng.random(n) < 0.8).astype("u1") if rng.random() < 0.5 else None
        if edges:
            data = _swapped_twin(rng, _mix_edges(rng, data))
        if op == "count*":
            aggs.append(O.agg("count", None, mask))
        elif op == "sum_moment":
            aggs.append(O.agg(op, data, mask, moment=int(rng.integers(0, 9 if edges else 5))))
        elif op in ("first", "last"):
            order = None
            if rng.random() < 0.7:
                odt = rng.choice(["f8", "i8", "i4", "u2", "f4"])
                order = rng.normal(0, 100, n).astype(odt) if np.dtype(odt).kind == "f" else rng.integers(0, 1000, n).astype(odt)
                if edges:
                    order = _mix_edges(rng, order)
            aggs.append(O.agg(op, data, mask, order=order))
        elif op == "nunique":
            sel = (rng.random(n) < 0.8).astype("u1") if rng.random() < 0.5 else None
            aggs.append(O.agg(op, data, mask, selection=sel, dropmissing=bool(rng.integers(0, 2)), dropnan=bool(rng.integers(0, 2))))
        else:
            aggs.append(O.agg(op, data, mask))
    return binners, aggs


# ---- exact per-cell references -------------------------------------------------------------------------------------------------
U = 2.0 ** -53
M64 = (1 << 64) - 1


def gamma(k):
    """the recursive-summation constant: |fl(sum) - sum| <= gamma(k) * sum|x_i| for k terms (Higham, Accuracy and Stability, 4.2)"""
    return k * U / (1 - k * U)


def _native(a):
    a = np.asarray(a)
    return a.astype(a.dtype.newbyteorder("=")) if a.dtype.byteorder not in ("=", "|") and a.dtype.byteorder != ("<" if np.little_endian else ">") else a


def used_rows(binners, a, n):
    """(flat cell per row, boolean: the row takes part in aggregator `a` = mask == 1 and the value is not NaN)"""
    from oracle import oracle as O
    idx, shapes = O.flat_indices(binners, n)
    use = np.ones(n, bool) if a["mask"] is None else (np.asarray(a["mask"])[:n] == 1)
    if a["data"] is not None:
        v = _native(a["data"])[:n]
        if v.dtype.kind == "f":
            use &= ~np.isnan(v)
    return idx.astype(np.int64), use, shapes


def pow_moment_int(b, m):
    """the device's power for integer grids (csrc/device_utils.cuh pow_moment / pow_moment_int), in IEEE double"""
    if m == 0:
        return 1.0
    if m == 4:
        b2 = b * b
        return b2 * b2
    r = b
    for _ in range(m - 1):
        r = r * b
    return r


def f64_to_i64_x86(x):
    return int(x) if -2.0 ** 63 <= x < 2.0 ** 63 else -(1 << 63)


def f64_to_u64_x86(x):
    if x >= 2.0 ** 63:
        return (f64_to_i64_x86(x - 2.0 ** 63) & M64) ^ (1 << 63)
    return f64_to_i64_x86(x) & M64


def int_moment_rule(binners, a, n):
    """integer sum_moment as the device computes it: per row the power in double, converted like the reference's x86-64 build
    (int64: out of range -> INT64_MIN; uint64: >= 2^64 -> 0), summed exactly mod 2^64.  Returns (expected grid, boolean grid:
    the cell's sum of |b^m| stays below 2^53, so the reference's double running sum is exact there and must agree bit for bit)."""
    from oracle import oracle as O
    idx, use, shapes = used_rows(binners, a, n)
    v = _native(a["data"])[:n]
    m = int(a["moment"])
    grid_dt = O.upcast(v.dtype)
    cells = int(np.prod(shapes))
    acc = [0] * cells
    mag = [0] * cells
    for c, x in zip(idx[use].tolist(), v[use].astype(object).tolist()):
        x = int(x)
        p = pow_moment_int(float(x), m)
        acc[c] += f64_to_i64_x86(p) if grid_dt == np.int64 else f64_to_u64_x86(p)
        mag[c] += abs(x) ** m
    want = np.array([s & M64 for s in acc], np.uint64).view(grid_dt)
    exact = np.array([s < (1 << 53) for s in mag])
    return want.reshape(shapes, order="F"), exact.reshape(shapes, order="F")


def float_sum_ok(binners, a, n, got):
    """floating sum / sum_moment: every cell of `got` within the recursive-summation bound of the exact sum of the powers
    (fractions), allowing for up to 4 roundings per power and for subnormal underflow.  Infinite powers decide the cell by IEEE
    rules; a cell whose sum of |powers| exceeds the largest double may also be +-inf / NaN.  Returns the first bad cell or None."""
    from fractions import Fraction
    idx, use, shapes = used_rows(binners, a, n)
    with np.errstate(invalid="ignore"):  # signalling NaN payloads; their rows do not take part
        v = _native(a["data"])[:n].astype(np.float64)
    m = 1 if a["op"] == "sum" else int(a["moment"])
    got = np.asarray(got).reshape(-1, order="F")
    cells = len(got)
    exact = [Fraction(0)] * cells
    mag = [Fraction(0)] * cells
    k = [0] * cells
    pinf, ninf = [False] * cells, [False] * cells
    with np.errstate(over="ignore", invalid="ignore"):
        p_float = np.power(v, m) if m else np.ones_like(v)
    for c, x, pf in zip(idx[use].tolist(), v[use].tolist(), p_float[use].tolist()):
        k[c] += 1
        if np.isinf(pf):
            (pinf if pf > 0 else ninf)[c] = True
            continue
        p = Fraction(x) ** m if m else Fraction(1)  # pow(x, 0) == 1 also for x = +-inf
        exact[c] += p
        mag[c] += abs(p)
    big = Fraction(np.finfo(np.float64).max)
    tiny = Fraction(2) ** -1074
    for c in range(cells):
        g = float(got[c])
        if pinf[c] and ninf[c]:
            ok = np.isnan(g)
        elif pinf[c] or ninf[c]:  # unless the finite powers overflowed to the other infinity first
            ok = g == (np.inf if pinf[c] else -np.inf) or (mag[c] > big and np.isnan(g))
        elif np.isfinite(g):
            bound = Fraction(gamma(k[c] + 4)) * mag[c] + 8 * k[c] * tiny
            ok = abs(Fraction(g) - exact[c]) <= bound
        else:
            ok = mag[c] > big
        if not ok:
            return c, g, k[c], pinf[c], ninf[c]
    return None


def zero_sign_rule(binners, a, n, want):
    """min / max of a float column as the device defines it: -0.0 < +0.0 (DESIGN §3).  Takes the oracle's grid and gives each cell
    whose extreme is a zero the sign the device rule picks from the zeros the cell saw."""
    idx, use, shapes = used_rows(binners, a, n)
    v = _native(a["data"])[:n]
    zeros = use & (v == 0)
    neg = np.zeros(int(np.prod(shapes)), bool)
    pos = np.zeros(int(np.prod(shapes)), bool)
    np.logical_or.at(neg, idx[zeros & np.signbit(v)], True)
    np.logical_or.at(pos, idx[zeros & ~np.signbit(v)], True)
    out = np.array(want, copy=True).reshape(-1, order="F")
    hit = out == 0
    pick = neg if a["op"] == "min" else pos
    out[hit & pick] = -0.0 if a["op"] == "min" else 0.0
    out[hit & ~pick] = 0.0 if a["op"] == "min" else -0.0
    return out.reshape(shapes, order="F")


def check_exact(binners, aggs, n, want, got, what=""):
    """the device's grids `got` against the oracle's `want` and, where DESIGN §3 says bits cannot match, against exact arithmetic:
    bit-exact for counts / integer sums / min / max / first-last / nunique; float min / max with the signed-zero rule; float sums
    and moments within the recursive-summation bound of the exact sum (the oracle too); integer moments by the device rule."""
    for k, (a, w, g) in enumerate(zip(aggs, want, got)):
        tag = (what, k, a["op"], a.get("moment"), None if a["data"] is None else np.asarray(a["data"]).dtype.str)
        kind = None if a["data"] is None else np.asarray(a["data"]).dtype.kind
        if a["op"] in ("sum", "sum_moment") and kind == "f":
            assert np.asarray(g).dtype == np.asarray(w).dtype and np.shape(g) == np.shape(w), tag
            assert float_sum_ok(binners, a, n, w) is None, ("oracle",) + tag
            assert float_sum_ok(binners, a, n, g) is None, tag + (float_sum_ok(binners, a, n, g),)
        elif a["op"] == "sum_moment":
            rule, exact = int_moment_rule(binners, a, n)
            assert same_bits(rule, g), tag
            assert same_bits(np.asarray(w)[exact], rule[exact]), ("oracle",) + tag
        elif a["op"] in ("min", "max") and kind == "f":
            assert same_bits(zero_sign_rule(binners, a, n, w), g), tag
        else:
            assert same_bits(w, g), tag


def edge_column(rng, dt, n, scale=10.0):
    """a column of dtype `dt` (either byte order): normal / small integer values with about a third replaced by edge values"""
    d = np.dtype(dt)
    if d.kind == "f":
        base = rng.normal(0, scale, n)
    elif d.kind == "b":
        base = rng.integers(0, 2, n)
    else:
        base = rng.integers(-50 if d.kind == "i" else 0, 100, n)
    return _mix_edges(rng, base.astype(d))
