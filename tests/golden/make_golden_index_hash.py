"""Generate tests/golden/index_hash_golden.npz: index_hash_<T> update / merge / lookup sequences and what the compiled, unmodified
reference classes (oracle/_ref superutils) return for them.

    python tests/golden/make_golden_index_hash.py [out.npz]

Every case stays inside the conditions where the reference is sequential (tests/index_hash_oracle.py): one update at start_index 0
(with NaN and masks), or several updates with increasing start_index and no NaN / null, merged in row order.  It covers the 11 dtypes,
nmaps 1 / 3 / 7, masks, NaN, several update calls, merges and every `out` width.  Only inputs and outputs are stored."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

DTYPES = ["bool", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
WIDTHS = ["int8", "int16", "int32", "int64"]


def _keys(rng, dtype, n, distinct):
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return rng.integers(0, 2, n).astype(bool)
    k = rng.integers(0, distinct, n)
    if dt.kind == "f":
        return (k * 0.5 - 7.25).astype(dt)
    if dt.kind == "i":
        return (k - distinct // 2).astype(dt)
    return k.astype(dt)


def cases():
    """name -> dict(dtype, nmaps, updates=[(keys, mask or None, start)], merges=[[(keys, mask, start)], ...], lookup, lookup_mask,
    dup_start).  Deterministic."""
    rng = np.random.default_rng(20261017)
    out = {}
    for dtype in DTYPES:
        for nmaps in (1, 3, 7):
            n = 300
            keys = _keys(rng, dtype, n, 60)
            mask = (rng.random(n) < 0.05).astype(np.uint8)
            if np.dtype(dtype).kind == "f":
                keys[rng.random(n) < 0.05] = np.nan
            look = np.concatenate([_keys(rng, dtype, 80, 90), keys[:20]])
            lmask = (rng.random(len(look)) < 0.1).astype(np.uint8)
            out[f"one_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=[(keys, mask, 0)], merges=[], lookup=look, lookup_mask=lmask, dup_start=1000)
            # several calls at increasing start_index, no NaN / null
            ups, start = [], 0
            for size in (50, 1, 120, 77):
                ups.append((_keys(rng, dtype, size, 40), None, start))
                start += size + int(rng.integers(0, 5))
            out[f"calls_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=ups, merges=[], lookup=_keys(rng, dtype, 100, 50), lookup_mask=None,
                                                 dup_start=-3)
            # merges in row order: each merged index holds later rows than everything before it
            parts, start = [], 0
            for size in (40, 70, 25):
                parts.append([(_keys(rng, dtype, size, 30), None, start)])
                start += size
            out[f"merge_{dtype}_{nmaps}"] = dict(dtype=dtype, nmaps=nmaps, updates=parts[0], merges=parts[1:], lookup=_keys(rng, dtype, 60, 35),
                                                 lookup_mask=None, dup_start=0)
    return out


def run(cls_of, case):
    """drive index_hash classes (reference or device) through a case: the results as a dict of arrays"""
    def build(updates):
        h = cls_of(case["dtype"])(case["nmaps"])
        for keys, mask, start in updates:
            if mask is None:
                h.update(keys, start)
            else:
                h.update(keys, mask, start)
        return h
    h = build(case["updates"])
    for m in case["merges"]:
        h.merge(build(m))
    look, lmask = case["lookup"], case["lookup_mask"]
    res = {}
    if lmask is None:
        res["map"] = np.asarray(h.map_index(look), np.int64)
        calls = {w: (lambda o: h.map_index(look, o)) for w in WIDTHS}
    else:
        res["map"] = np.asarray(h.map_index_masked(look, lmask), np.int64)
        calls = {w: (lambda o: h.map_index_masked(look, lmask, o)) for w in WIDTHS}
    for w in WIDTHS:
        o = np.zeros(len(look), w)
        res["unknown_" + w] = np.array(bool(calls[w](o)))
        res["map_" + w] = o
    left, right = h.map_index_duplicates(look, case["dup_start"])
    res["dup_left"], res["dup_right"] = np.asarray(left, np.int64), np.asarray(right, np.int64)
    res["scalars"] = np.array([len(h), h.count, h.has_duplicates, h.nan_count, h.null_count], np.int64)
    return res


def flatten(name, case, res):
    flat = {}
    for j, (keys, mask, start) in enumerate(case["updates"]):
        flat[f"{name}/u{j}_keys"], flat[f"{name}/u{j}_start"] = keys, np.array(start)
        if mask is not None:
            flat[f"{name}/u{j}_mask"] = mask
    for i, m in enumerate(case["merges"]):
        for j, (keys, _, start) in enumerate(m):
            flat[f"{name}/m{i}_{j}_keys"], flat[f"{name}/m{i}_{j}_start"] = keys, np.array(start)
    flat[f"{name}/lookup"] = case["lookup"]
    if case["lookup_mask"] is not None:
        flat[f"{name}/lookup_mask"] = case["lookup_mask"]
    for k, v in res.items():
        flat[f"{name}/out_{k}"] = v
    return flat


def load(path):
    """the golden file back as {name: (case, reference results)}"""
    z = np.load(path)
    names = sorted({k.split("/")[0] for k in z.files})
    dtypes_nmaps = {n: (n.split("_")[1], int(n.split("_")[2])) for n in names}
    out = {}
    for n in names:
        dtype, nmaps = dtypes_nmaps[n]
        ups, j = [], 0
        while f"{n}/u{j}_keys" in z.files:
            ups.append((z[f"{n}/u{j}_keys"], z[f"{n}/u{j}_mask"] if f"{n}/u{j}_mask" in z.files else None, int(z[f"{n}/u{j}_start"])))
            j += 1
        merges, i = [], 0
        while f"{n}/m{i}_0_keys" in z.files:
            merges.append([(z[f"{n}/m{i}_0_keys"], None, int(z[f"{n}/m{i}_0_start"]))])
            i += 1
        case = dict(dtype=dtype, nmaps=nmaps, updates=ups, merges=merges, lookup=z[f"{n}/lookup"],
                    lookup_mask=z[f"{n}/lookup_mask"] if f"{n}/lookup_mask" in z.files else None,
                    dup_start={"one": 1000, "calls": -3, "merge": 0}[n.split("_")[0]])
        res = {k.split("/out_")[1]: z[k] for k in z.files if k.startswith(n + "/out_")}
        out[n] = (case, res)
    return out


def main():
    from oracle import ref_driver
    su = ref_driver.modules()[1]
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "index_hash_golden.npz")
    flat = {}
    for name, case in cases().items():
        flat.update(flatten(name, case, run(lambda dt: getattr(su, "index_hash_" + dt), case)))
    from make_golden_edges import save
    save(path, flat)
    print(f"wrote {path}: {len(cases())} cases")


if __name__ == "__main__":
    main()
