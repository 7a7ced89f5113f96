"""Generate tests/golden/binstats_golden.npz from the COMPILED, UNMODIFIED reference (oracle/_ref).

Run in the build container (where /root/reference exists and `make -C oracle ref` has been run):

    python tests/golden/make_golden.py

Every case stores its inputs and the reference's outputs, so the fixtures pin both the oracle (CPU, `-m "not gpu"`) and
the CUDA path (`-m gpu`) without needing the reference at test time.  Cases mirror what the reference's own tests pin:
tests/agg_test.py:150-158, :171-180 (exact grids), :8-48 (sum), :257-281 (big-endian / strided), :395-402 (upcast),
tests/internal/superagg_tests.py:49-120 (scalar-binner count vectors, with the `threads` ctor argument added),
tests/internal/hash_test.py:78-150 (ordered_set incl. null/NaN ordinals and map_ordinal dtype).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402
from oracle import ref_driver as R  # noqa: E402


def add_case(out, name, binners, aggs, n):
    """run the compiled reference on one (binners, aggs) problem; store inputs and outputs as `name/<field>` arrays in `out`"""
    res = R.binby(binners, aggs, n)
    c = {"n": n, "nb": len(binners), "na": len(aggs)}
    for i, b in enumerate(binners):
        c[f"b{i}_kind"] = b["kind"]
        c[f"b{i}_data"] = b["data"]
        c[f"b{i}_dtype"] = b["data"].dtype.str  # npz drops byte order
        if b["mask"] is not None:
            c[f"b{i}_mask"] = b["mask"]
        for k in ("vmin", "vmax", "bins", "count", "min_value", "allow_other", "invert"):
            if k in b:
                c[f"b{i}_{k}"] = b[k]
    for k, (a, r) in enumerate(zip(aggs, res)):
        c[f"a{k}_op"] = a["op"]
        if a["data"] is not None:
            c[f"a{k}_data"] = a["data"]
            c[f"a{k}_dtype"] = a["data"].dtype.str
        if a["mask"] is not None:
            c[f"a{k}_mask"] = a["mask"]
        if a.get("moment") is not None:
            c[f"a{k}_moment"] = a["moment"]
        if a.get("order") is not None:
            c[f"a{k}_order"] = a["order"]
        if a.get("selection") is not None:
            c[f"a{k}_selection"] = a["selection"]
        if a["op"] == "nunique":
            c[f"a{k}_drop"] = np.array([a["dropmissing"], a["dropnan"]])
        if np.ma.isMaskedArray(r):
            c[f"a{k}_result"] = np.asarray(r.data)
            c[f"a{k}_result_mask"] = np.ma.getmaskarray(r)
        else:
            c[f"a{k}_result"] = np.asarray(r)
    for k, v in c.items():
        out[f"{name}/{k}"] = np.asarray(v)


def cases():
    rng = np.random.default_rng(20260922)
    out = {}

    def add(name, binners, aggs, n):
        add_case(out, name, binners, aggs, n)

    # KATs of the reference test-suite
    x = np.array([-1, -2, 0.5, 1.5, 4.5, 5], dtype="f8")
    add("kat_count_1d", [O.scalar(x, 0, 5, 5)], [O.agg("count")], 6)
    xi = np.array([-1, -2, 0, 1, 4, 5], dtype="i8")
    add("kat_count_1d_ordinal", [O.ordinal(xi, 5, 0)], [O.agg("count")], 6)
    # superagg_tests.py:49-59 style: x = arange(10), 5 bins over [0, 10)... plus weights
    x = np.arange(10, dtype="f8")
    y = x ** 2
    add("kat_arange_sum", [O.scalar(x, 0, 10, 5)], [O.agg("count"), O.agg("sum", y), O.agg("min", y), O.agg("max", y)], 10)
    # big-endian + strided source (agg_test.py:257-281)
    xb = np.arange(20, dtype=">f8")
    ys = np.arange(40, dtype="f8")[::2] ** 2
    add("kat_bigendian_strided", [O.scalar(xb, 0, 20, 4)], [O.agg("sum", np.ascontiguousarray(ys)), O.agg("count", xb)], 20)
    # upcast (agg_test.py:395-402)
    add("kat_upcast", [O.scalar(x, 0, 10, 2)], [O.agg("sum", np.arange(10, dtype="i1") * 12), O.agg("sum", np.arange(10, dtype="f4") + 0.1),
                                                O.agg("sum", np.arange(10, dtype="u2") * 6000)], 10)
    # headline-shaped sample: 2-D 1024^2 on fp32 gaussians with limits [-3, 3], NaNs injected
    n = 50_000
    gx, gy, gz = (rng.normal(0, 1, n).astype("f4") for _ in range(3))
    gx[::997] = np.nan
    add("headline_2d_f32", [O.scalar(gx, -3, 3, 1024), O.scalar(gy, -3, 3, 1024)], [O.agg("count"), O.agg("sum", gz), O.agg("count", gz)], n)
    # 3-D fp64 mean+std primitives (config 3 shape, tiny)
    n = 20_000
    a, b, c, v = (rng.normal(0, 1, n) for _ in range(4))
    add("c3_3d_f64", [O.scalar(a, -3, 3, 16), O.scalar(b, -3, 3, 16), O.scalar(c, -3, 3, 16)],
        [O.agg("count", v), O.agg("sum", v), O.agg("sum_moment", v, moment=2)], n)
    # masks + selections + every integer dtype through the ordinal binner
    n = 3000
    for dt in ("i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?"):
        if dt == "?":
            codes = rng.integers(0, 2, n).astype(dt)
        else:
            codes = rng.integers(-2 if np.dtype(dt).kind == "i" else 0, 9, n).astype(dt)
        vals = rng.integers(-100, 100, n).astype("i4")
        add(f"ordinal_{np.dtype(dt).name}", [O.ordinal(codes, 6, 1, bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), mask=rng.random(n) < 0.1)],
            [O.agg("count", None, (rng.random(n) < 0.7).astype("u1")), O.agg("sum", vals), O.agg("min", vals), O.agg("max", vals)], n)
    # first / last with an order column (single chunk <= 1024 rows so the mask-offset quirk is not in play)
    n = 1000
    fx = rng.uniform(0, 4, n)
    fv = rng.normal(0, 1, n)
    fo = rng.integers(0, 40, n).astype("i8")
    add("first_last", [O.scalar(fx, 0, 4, 4)], [O.agg("first", fv, None, order=fo), O.agg("last", fv, None, order=fo), O.agg("first", fv, None)], n)
    # AggNUnique (src/agg_nunique.cpp; tests/agg_test.py:294-333): the float KAT of the reference test, then random cells with
    # several NaN / null rows each (dropmissing / dropnan subtract ROW counts), selections, every dtype family, byte-swapped input
    kx = np.array([0, 0, 0, 0, 0, 1, 1, 1, 2], dtype="f8")
    ks = np.array([1.2, 1.2, 2.5, 3.7, np.nan, 3.7, 4.8, 3.7, 1.2])
    add("nunique_kat", [O.scalar(kx, 0, 3, 3)], [O.agg("nunique", ks), O.agg("nunique", ks, dropnan=True)], 9)
    ky = np.array([1, 1, 0, 1, 0, 0, 0, 1, 1], dtype="u1")
    add("nunique_kat_filtered", [O.scalar(kx, 0, 3, 3)], [O.agg("nunique", ks, selection=(ky == 0).astype("u1"))], 9)
    n = 3000
    gx = rng.uniform(0, 5, n)
    gy = rng.integers(0, 4, n).astype("i4")
    for dt in ("f8", "f4", "i8", "i2", "u1", "?", ">f8", ">i4"):
        d = np.dtype(dt)
        if d.kind == "f":
            v = (rng.integers(-6, 6, n) * 0.5).astype(d)
            v[rng.random(n) < 0.1] = np.nan
            v[rng.random(n) < 0.05] = -0.0
        elif d.kind == "b":
            v = rng.integers(0, 2, n).astype(d)
        else:
            v = rng.integers(0 if d.kind == "u" else -8, 9, n).astype(d)
        valid = (rng.random(n) < 0.85).astype("u1")
        sel = (rng.random(n) < 0.7).astype("u1")
        add("nunique_" + d.name + ("_be" if dt.startswith(">") else ""), [O.scalar(gx, 0, 5, 6), O.ordinal(gy, 4)],
            [O.agg("nunique", v), O.agg("nunique", v, valid, dropmissing=True), O.agg("nunique", v, valid, selection=sel, dropnan=True),
             O.agg("nunique", v, valid, selection=sel, dropmissing=True, dropnan=True), O.agg("count", v)], n)
    return out


def hash_cases():
    rng = np.random.default_rng(7)
    out = {}
    for dt in ("float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool"):
        d = np.dtype(dt)
        for nmaps in (1, 3):
            n = 2000
            if d.kind == "f":
                k = rng.integers(-20, 50, n).astype(d) * 0.5
                k[rng.random(n) < 0.05] = np.nan
            elif d.kind == "b":
                k = rng.integers(0, 2, n).astype(d)
            else:
                k = rng.integers(max(np.iinfo(d).min, -1000), min(np.iinfo(d).max, 1000), n).astype(d)
            m = rng.random(n) < 0.03
            s = R.ordered_set(d, nmaps)
            vals, mi = s.update(k, m, 0, 1024 * 1024, 4 * 1024 * 1024, True)
            name = f"set_{dt}_{nmaps}"
            out[f"{name}/keys"] = k
            out[f"{name}/mask"] = m
            out[f"{name}/values"] = np.asarray(vals)
            out[f"{name}/map_index"] = np.asarray(mi)
            out[f"{name}/key_array"] = np.asarray(s.key_array())
            out[f"{name}/offsets"] = np.asarray(s.offsets())
            out[f"{name}/map_ordinal"] = np.asarray(s.map_ordinal(k))
            out[f"{name}/null_nan"] = np.array([s.null_index, s.nan_index, s.null_count, s.nan_count])
    out["hash64/in"] = np.array([1, 2, 0, 2 ** 63, 123456789], dtype="u8")
    _, su = R.modules()
    out["hash64/out"] = np.array([su.hash(int(v)) for v in out["hash64/in"]], dtype="u8")
    return out


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    data = cases()
    data.update(hash_cases())
    np.savez_compressed(os.path.join(here, "binstats_golden.npz"), **data)
    print("wrote", len(data), "arrays,", os.path.getsize(os.path.join(here, "binstats_golden.npz")) // 1024, "KiB")
