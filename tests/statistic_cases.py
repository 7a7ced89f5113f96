"""Seeded random cases for the legacy statistics (csrc/statistic.cu): every dtype, both byte orders, masked blocks, 0-3 binby
dimensions, edges on and off, all seven ops, COV with 1-5 weights and lists of selections."""
import numpy as np

from statistic_oracle import ADD1, COUNT, COV, FIRST, MIN_MAX, MOMENTS_01, MOMENTS_012

DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"]
OPS = [ADD1, COUNT, MIN_MAX, MOMENTS_01, MOMENTS_012, COV, FIRST]


def column(rng, dtype, n, lo=-4.0, hi=4.0):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        a = rng.uniform(lo, hi, n).astype(dt)
        special = rng.random(n)
        a[special < 0.03] = np.nan
        a[(special >= 0.03) & (special < 0.04)] = 0.0
        a[(special >= 0.04) & (special < 0.05)] = -0.0
        a[(special >= 0.05) & (special < 0.055)] = np.inf
        a[(special >= 0.055) & (special < 0.06)] = -np.inf
        a[(special >= 0.06) & (special < 0.07)] = lo  # on a bin edge
        return a
    if dt.kind == "b":
        return rng.random(n) < 0.5
    info = np.iinfo(dt)
    a = rng.integers(max(info.min, -5), min(info.max, 5), n, endpoint=True).astype(dt)
    big = rng.random(n) < 0.05  # values that float32 (or float64) cannot hold exactly
    a[big] = rng.integers(info.min, info.max, int(big.sum()), endpoint=True, dtype=dt)
    return a


def random_case(rng, n=3000):
    op = OPS[rng.integers(len(OPS))]
    nd = int(rng.integers(0, 4))
    nw = {ADD1: int(rng.integers(0, 2)), COV: int(rng.integers(1, 6)), FIRST: 2}.get(op, 1)
    if nd == 0 and nw == 0:
        nw = 1
    edges = bool(rng.random() < 0.5) and nd > 0
    dtypes = [DTYPES[rng.integers(len(DTYPES))] for _ in range(nd + nw)]
    if rng.random() < 0.3:  # a float column steers the compute class
        dtypes[int(rng.integers(len(dtypes)))] = ["float32", "float64"][rng.integers(2)]
    swap = rng.random() < 0.25  # all blocks byte-swapped (the reference rejects a mix of orders in one call)
    cols = []
    for dt in dtypes:
        a = column(rng, dt, n)
        if swap and np.dtype(dt).itemsize > 1:
            a = a.astype(np.dtype(dt).newbyteorder(">" if np.little_endian else "<"))
        if rng.random() < 0.25:
            a = np.ma.array(a, mask=rng.random(n) < 0.1)
        cols.append(a)
    sizes = [int(rng.choice([1, 3, 7, 16, 100])) + (3 if edges else 0) for _ in range(nd)]
    minima = [float(rng.uniform(-4, 0)) for _ in range(nd)]
    maxima = [float(m + rng.uniform(0.5, 6)) for m in minima]
    nsel = int(rng.integers(1, 4))
    selections = [None if rng.random() < 0.3 else rng.random(n) < 0.6 for _ in range(nsel)]
    return dict(binby=cols[:nd], weights=cols[nd:], selections=selections, op=op, sizes=sizes, minima=minima, maxima=maxima, edges=edges)
