"""A numpy restatement of the legacy statistics (vaexfast statisticNd, src/vaexfast.cpp:1061-1278, driven by TaskPartStatistic.process,
vaex/cpu.py:510-616) — the checker for csrc/statistic.cu — and the same driver around the compiled, unmodified vaexfast
(oracle/_ref) that pins the restatement bit for bit.

``process(binby, weights, selections, op, sizes, minima, maxima, edges, chunk, impl)`` returns the grid (nselections, *sizes,
fields) BEFORE the op's reduce, accumulated chunk by chunk in row order like one reference thread."""
import numpy as np

ADD1, COUNT, MIN_MAX, MOMENTS_01, MOMENTS_012, COV, FIRST = range(7)


def fields(op, nweights):
    return {ADD1: 1, COUNT: 1, MIN_MAX: 2, MOMENTS_01: 2, MOMENTS_012: 3, FIRST: 2}.get(op, 2 * nweights + 2 * nweights**2)


def init_grid(op, shape):
    grid = np.zeros(shape, np.float64)
    if op == MIN_MAX:
        grid[..., 0], grid[..., 1] = np.inf, -np.inf
    if op == FIRST:
        grid[..., 0], grid[..., 1] = np.nan, np.inf
    return grid


def compute_dtype(dtypes):
    """vaex/cpu.py:527-541 -> the numpy class every block is cast to"""
    dtype = np.result_type(*dtypes)
    if dtype.str in ">f8 <f8 =f8" or dtype.str in ">i8 <i8 =i8":
        return np.dtype(np.float64)
    return np.dtype(np.float32)


def _native(a):
    return a.astype(a.dtype.newbyteorder("=")) if a.dtype.byteorder not in "=|" else a


def statistic_nd(blocks, weights, grid, minima, maxima, op, edges):
    """statisticNd on blocks already cast to the class T (numpy arrays of T, native order): accumulates into `grid` (*sizes, fields)"""
    T = (blocks + weights)[0].dtype.type if blocks or weights else np.float32
    sizes = grid.shape[:-1]
    nd = len(blocks)
    n = len(blocks[0]) if blocks else (len(weights[0]) if weights else 0)
    idx = np.zeros(n, np.int64)
    inside = np.ones(n, bool)
    stride = 1
    strides = [0] * nd
    for d in range(nd - 1, -1, -1):
        strides[d] = stride
        stride *= sizes[d]
    with np.errstate(all="ignore"):
        for d in range(nd):
            lo, hi = T(minima[d]), T(maxima[d])
            scale = T(1) / (hi - lo)
            scaled = (blocks[d] - lo) * scale
            size = sizes[d]
            if edges:
                inner = (scaled.astype(np.float64) * (size - 3))
                inner = np.where(np.isfinite(inner), inner, 0).astype(np.int64) + 2
                sub = np.where(scaled != scaled, 0, np.where(scaled < 0, 1, np.where(scaled >= 1, size - 1, inner)))
            else:
                ok = (scaled >= 0) & (scaled < 1)
                inside &= ok
                prod = scaled * T(size) if nd == 2 else scaled.astype(np.float64) * size
                sub = np.where(ok, prod, 0).astype(np.int64)
            idx += strides[d] * sub
    rows = np.nonzero(inside)[0]
    cell = idx[rows]
    flat = grid.reshape(-1, grid.shape[-1])
    w = [np.asarray(x, np.float64)[rows] for x in weights]
    if op == ADD1:
        np.add.at(flat[:, 0], cell, 1.0)
    elif op == COUNT:
        np.add.at(flat[:, 0], cell[~np.isnan(w[0])], 1.0)
    elif op in (MOMENTS_01, MOMENTS_012):
        ok = ~np.isnan(w[0])
        np.add.at(flat[:, 0], cell[ok], 1.0)
        np.add.at(flat[:, 1], cell[ok], w[0][ok])
        if op == MOMENTS_012:
            np.add.at(flat[:, 2], cell[ok], w[0][ok] * w[0][ok])
    elif op == MIN_MAX:
        ok = ~np.isnan(w[0])
        c, v = cell[ok], w[0][ok]
        for k, fn in ((0, np.minimum), (1, np.maximum)):
            before = flat[:, k].copy()
            fn.at(flat[:, k], c, v)
            # strict compares keep the zero that arrived first (or the one already there)
            zero = np.nonzero(flat[:, k] == 0)[0]
            for z in zero:
                if before[z] == 0:
                    flat[z, k] = before[z]
                    continue
                first = np.nonzero((c == z) & (v == 0))[0][0]
                flat[z, k] = v[first]
    elif op == COV:
        N = len(w)
        for i in range(N):
            oki = ~np.isnan(w[i])
            np.add.at(flat[:, i], cell[oki], 1.0)
            np.add.at(flat[:, N + i], cell[oki], w[i][oki])
            for j in range(i, N):
                both = oki & ~np.isnan(w[j])
                a, b = 2 * N + j + i * N, 2 * N + i + j * N
                np.add.at(flat[:, a], cell[both], 1.0)
                np.add.at(flat[:, 2 * N + N * N + j + i * N], cell[both], w[i][both] * w[j][both])
                flat[:, b] = flat[:, a]
                flat[:, 2 * N + N * N + i + j * N] = flat[:, 2 * N + N * N + j + i * N]
    elif op == FIRST:
        order = w[1]
        ok = order < np.inf
        pos = np.nonzero(ok)[0]
        best = {}  # strict `order < best`: NaN and +inf never win, ties keep the earliest row
        for p in pos:
            c = cell[p]
            if order[p] < (best[c][1] if c in best else flat[c, 1]):
                best[c] = (w[0][p], order[p])
        for c, (v, o) in best.items():
            flat[c, 0], flat[c, 1] = v, o
    return grid


def _vaexfast_nd(blocks, weights, grid, minima, maxima, op, edges):
    from oracle import ref_driver
    vf = ref_driver.vaexfast()
    fn = vf.statisticNd_f8 if (blocks + weights)[0].dtype.itemsize == 8 else vf.statisticNd_f4
    fn(list(blocks), list(weights) or None, grid, [float(v) for v in minima], [float(v) for v in maxima], op, int(edges))
    return grid


def process(binby, weights, selections, op, sizes, minima, maxima, edges=False, chunk=None, impl="oracle"):
    """TaskPartStatistic.process over chunks of `chunk` rows: masked rows (any block) dropped from every selection, each selection
    filtered by its mask, every block cast to the compute class; impl = "oracle" (statistic_nd) or "vaexfast" (compiled reference)"""
    nd_fn = statistic_nd if impl == "oracle" else _vaexfast_nd
    n = len((list(binby) + list(weights))[0])
    chunk = chunk or max(n, 1)
    grid = init_grid(op, (len(selections),) + tuple(sizes) + (fields(op, len(weights)),))
    for i1 in range(0, n, chunk):
        blocks = [b[i1:i1 + chunk] for b in list(binby) + list(weights)]
        masks = [np.ma.getmaskarray(b) for b in blocks if np.ma.isMaskedArray(b)]
        blocks = [np.asarray(b.data if np.ma.isMaskedArray(b) else b) for b in blocks]
        T = compute_dtype([b.dtype for b in blocks])
        mask = None
        if masks:
            mask = np.logical_or.reduce(masks)
            blocks = [b[~mask] for b in blocks]
        for s, sel in enumerate(selections):
            sb = blocks
            if sel is not None:
                m = np.asarray(sel[i1:i1 + chunk], bool)
                if mask is not None:
                    m = m[~mask]
                sb = [b[m] for b in blocks]
            if impl == "oracle":
                sb = [_native(b).astype(T) for b in sb]
            else:  # the reference: mixed byte orders are made native, then as_flat_array (vaex/utils.py:691-695)
                little = [b.dtype.byteorder in "<=|" for b in sb]
                if not (all(little) or not any(little)):
                    sb = [_native(b) for b in sb]
                sb = [b if (b.dtype.type == T.type and b.strides[0] == 8) else b.astype(T) for b in sb]
                if len({b.dtype.byteorder in "<=|" for b in sb}) > 1:  # statisticNd_ raises on this mix; the values are the same
                    sb = [_native(b) for b in sb]
            if len(sb) == 0:
                grid[s][..., 0] += len(sel[i1:i1 + chunk]) if sel is None else np.sum(sel[i1:i1 + chunk])
                continue
            nd_fn(sb[:len(binby)], sb[len(binby):], grid[s], minima, maxima, op, edges)
    return grid
