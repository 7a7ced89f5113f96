"""tests/golden/agglist_string_golden.npz (tests/golden/make_golden_agglist_string.py), shared by the CPU and GPU tests of
AggList_string_int64: per setup the rows (string buffers, data mask, binner columns, the bin() call ranges) and per case the arrow
buffers the compiled reference returned (buffers the file stores once for several cases are resolved here)."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agglist_string_golden.npz")
SETUPS = ("ord", "ord_scalar", "one_cell", "sparse")


def load():
    z = np.load(PATH, allow_pickle=False)
    setups = {}
    for name in SETUPS:
        s = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/") and k.count("/") == 1}
        binners = []
        for i in range(int(s["nbinners"])):
            arg = s[f"b{i}_arg"]
            binners.append((str(s[f"b{i}_kind"]), s[f"b{i}_data"], int(arg[0]) if str(s[f"b{i}_kind"]) == "ordinal" else tuple(arg)))

        def field(case, f):  # a buffer equal to an earlier case's is stored once, the later case names that case
            key = f"{name}/{case}/{f}"
            return z[key] if key in z.files else field(str(z[key + "_same_as"]), f)

        cases = {}
        for case in sorted({k.split("/")[1] for k in z.files if k.startswith(name + "/") and k.count("/") == 2}):
            cases[case] = dict(masked=case.startswith("masked"), dropnan="dropnan1" in case, dropnull="dropnull1" in case,
                               **{f: field(case, f) for f in ("list_offsets", "str_offsets", "str_bytes", "str_valid")})
        setups[name] = dict(n=int(s["n"]), calls=[tuple(c) for c in s["calls"].tolist()], offsets=s["offsets"], bytes=s["bytes"], nulls=s["nulls"],
                            valid=s["valid"], binners=binners, cases=cases)
    return setups


def strings_of(setup):
    off, by, nulls = setup["offsets"], setup["bytes"], setup["nulls"]
    return [None if nulls[i] else bytes(by[off[i]:off[i + 1]]).decode("utf8") for i in range(len(off) - 1)]


def flat_cells(setup):
    """the flat grid cell of every row (first binner fastest) and the cell count, from the oracle's binner restatement"""
    from oracle import oracle as O
    bs = []
    for kind, data, arg in setup["binners"]:
        bs.append(O.ordinal(data, arg, 0) if kind == "ordinal" else O.scalar(data, arg[0], arg[1], int(arg[2])))
    cells = O.flat_indices(bs, setup["n"])[0].astype(np.int64)
    ncells = 1
    for b in bs:
        ncells *= O.binner_shape(b)
    return cells, ncells
