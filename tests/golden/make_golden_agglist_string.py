"""Generate tests/golden/agglist_string_golden.npz from the COMPILED, UNMODIFIED reference (oracle/_ref/superagg*.so):
AggList_string_int64 (src/agg_list.cpp:122-222), fed in 2-3 bin() calls whose cuts are not on a 1024-row boundary, for the four
dropnan / dropnull combinations, with and without a data mask (which the reference never reads).  Run where /root/reference exists:

    make -C oracle ref && python tests/golden/make_golden_agglist_string.py

The strings reach the reference as its own StringList64 through oracle/ref_strlist_shim.cpp (its StringSequence / StringList64
registered with pybind11; superagg accepts them in set_data), and get_result() hands (offsets, StringList64) to
vaex.arrow.convert.list_from_arrays, which vaex cannot provide here: a stub module with that one function stands in, and the shim
turns the StringList64 back into buffers.

Setups (binners over the same rows): `ord` one ordinal binner with out-of-range codes; `ord_scalar` ordinal x scalar (NaN keys);
`one_cell` every row in one cell; `sparse` 2000 categories for 300 rows, most cells empty.  Strings: a vocabulary with the empty
string, multi-byte UTF-8 and strings over 64 B, a few over 4 KB, and nulls.

Per case ('<setup>/<plain|masked>_dropnan<0|1>_dropnull<0|1>') the four arrow buffers the reference returned.  A buffer equal to
the same buffer of an earlier case of the setup (the data mask and dropnan change nothing) is stored once: the later case holds
'<field>_same_as' = the earlier case's name instead (tests/agglist_string_cases.py resolves it)."""
import importlib
import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_driver as R  # noqa: E402


def _stub_vaex():
    vaex = types.ModuleType("vaex")
    arrow = types.ModuleType("vaex.arrow")
    convert = types.ModuleType("vaex.arrow.convert")
    convert.list_from_arrays = lambda offsets, values: (np.array(offsets), values)
    vaex.arrow, arrow.convert = arrow, convert
    sys.modules.update({"vaex": vaex, "vaex.arrow": arrow, "vaex.arrow.convert": convert})


def _shim():
    sys.path.insert(0, R._REF)
    try:
        return importlib.import_module("strlist_shim")
    finally:
        sys.path.remove(R._REF)


def strings(rnd, n, null_rate=0.1):
    alphabet = "abcdefghijklmnopqrstuvwxyz0123456789 _-äß€😀"
    vocab = [""] + ["".join(rnd.choice(alphabet) for _ in range(rnd.choice([1, 2, 3, 5, 8, 15, 16, 17, 31, 33, 65, 70]))) for _ in range(200)]
    out = [rnd.choice(vocab) if rnd.random() >= null_rate else None for _ in range(n)]
    for i in rnd.sample(range(n), min(3, n)):  # a few strings over 4 KB, made of vocabulary words (they compress)
        s = ""
        while len(s.encode()) <= 4096 + rnd.randrange(2000):
            s += rnd.choice(vocab)
        out[i] = s
    return out


def setups(rnd, rng):
    n = 2000
    yield "ord", n, (n // 3 + 17, 2 * n // 3 + 5), [("ordinal", rng.integers(-1, 11, n).astype("i4"), 9)]
    y = rng.uniform(-0.2, 1.2, n)
    y[rng.random(n) < 0.05] = np.nan
    yield "ord_scalar", n, (1777,), [("ordinal", rng.integers(0, 5, n).astype("i8"), 5), ("scalar", y, (0.0, 1.0, 4))]
    yield "one_cell", n, (700, 1500), [("ordinal", np.full(n, 3, "i4"), 9)]
    m = 300
    yield "sparse", m, (101, 257), [("ordinal", rng.integers(0, 2000, m).astype("i8"), 2000)]


def main():
    _stub_vaex()
    sa, _ = R.modules()
    shim = _shim()
    rnd = random.Random(20261015)
    rng = np.random.default_rng(1015)
    out = {}
    for name, n, cuts, binners in setups(rnd, rng):
        strs = strings(rnd, n)
        off, by, nulls = R.pack_strings(strs)
        valid = (rng.random(n) < 0.7).astype("u1")  # the data mask: the reference stores it and never reads it
        bounds = [0, *cuts, n]
        calls = list(zip(bounds[:-1], bounds[1:]))
        out[f"{name}/n"] = np.array(n)
        out[f"{name}/calls"] = np.array(calls, np.int64)
        out[f"{name}/offsets"], out[f"{name}/bytes"], out[f"{name}/nulls"], out[f"{name}/valid"] = off, by, nulls, valid
        out[f"{name}/nbinners"] = np.array(len(binners))
        for i, (kind, data, arg) in enumerate(binners):
            out[f"{name}/b{i}_kind"], out[f"{name}/b{i}_data"] = np.array(kind), data
            out[f"{name}/b{i}_arg"] = np.array(arg if kind == "scalar" else (arg,), np.float64)
        seen = {}
        for masked in (False, True):
            for dropnan in (False, True):
                for dropnull in (False, True):
                    bs = []
                    for kind, data, arg in binners:
                        if kind == "ordinal":
                            bs.append(getattr(sa, "BinnerOrdinal_" + data.dtype.name)(1, "x", arg, 0, False, False))
                        else:
                            bs.append(getattr(sa, "BinnerScalar_" + data.dtype.name)(1, "y", arg[0], arg[1], int(arg[2])))
                    g = sa.Grid(bs)
                    a = sa.AggList_string_int64(g, 1, 1, dropnan, dropnull)
                    keep = []
                    for i1, i2 in calls:
                        for b, (_, data, _) in zip(bs, binners):
                            block = np.ascontiguousarray(data[i1:i2])
                            keep.append(block)
                            b.set_data(0, block)
                        coff = off[i1:i2 + 1] - off[i1]
                        sl = shim.make(np.ascontiguousarray(coff), np.ascontiguousarray(by[off[i1]:off[i2]]), np.ascontiguousarray(nulls[i1:i2]))
                        keep.append(sl)
                        a.set_data(0, sl, 0)
                        if masked:
                            ms = np.ascontiguousarray(valid[i1:i2])
                            keep.append(ms)
                            a.set_data_mask(0, ms)
                        else:
                            a.clear_data_mask(0)
                        g.bin(0, [a], i2 - i1)
                    list_offsets, sl = a.get_result()
                    soff, sby, sval = shim.buffers(sl)
                    case = f"{'masked' if masked else 'plain'}_dropnan{int(dropnan)}_dropnull{int(dropnull)}"
                    fields = dict(list_offsets=np.asarray(list_offsets, np.int64), str_offsets=np.asarray(soff), str_bytes=np.asarray(sby),
                                  str_valid=np.asarray(sval))
                    for field, value in fields.items():
                        # an array equal to the same field of an earlier case of the setup is stored once: the file names that case
                        same = next((c for c, f in seen.items() if np.array_equal(f[field], value)), None)
                        if same is None:
                            out[f"{name}/{case}/{field}"] = value
                        else:
                            out[f"{name}/{case}/{field}_same_as"] = np.array(same)
                    seen[case] = fields
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "agglist_string_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == "__main__":
    main()
