"""Generate tests/golden/set_edges_golden.npz from the COMPILED reference's ordered_set_<T> (src/hash_primitives.hpp) over the
edge corpus of tests/set_cases.py (without -0.0, whose treatment depends on the reference's table size).  Run where
/root/reference exists:

    make -C oracle ref && python tests/golden/make_golden_set_edges.py

Per case '<dtype>_<nmaps>_<sequence>': the update calls (keys, mask, (start_index, return_values)), what the calls with
return_values returned, the final key array as raw bits (the NaN slot zeroed), shard offsets, (nan_count, nan_index),
(null_count, null_index) -- index 0 when the count is 0 --, and map_ordinal / isin of the corpus queries.  Plus 'merge_*': the
reference's merge with a NaN on either side."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import set_cases as S  # noqa: E402
from oracle import ref_driver as R  # noqa: E402


def bits(a):
    a = np.asarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


GOLDEN_ROWS = 500  # filler rows per corpus column: the edge values are all there, the file stays small


def cases():
    out = {}
    for dtype in S.DTYPES:
        q = S.queries(dtype, zeros=False)
        for nmaps in (1, 3, 257):
            for name, calls in S.sequences(dtype, zeros=False, n=GOLDEN_ROWS):
                key = f"{dtype}_{nmaps}_{name}"
                s = R.ordered_set(dtype, nmaps)
                out[f"{key}/dtype"], out[f"{key}/nmaps"], out[f"{key}/ncalls"] = np.array(dtype), np.array(nmaps), np.array(len(calls))
                for i, c in enumerate(calls):
                    kw = dict(start_index=c["start_index"], return_values=c["return_values"])
                    out[f"{key}/c{i}_keys"] = c["keys"]
                    out[f"{key}/c{i}_opts"] = np.array([c["start_index"], int(c["return_values"])])
                    if c["mask"] is not None:
                        out[f"{key}/c{i}_mask"] = c["mask"]
                        r = s.update(c["keys"], np.ascontiguousarray(c["mask"], bool), **kw)
                    else:
                        r = s.update(c["keys"], **kw)
                    if c["return_values"]:
                        out[f"{key}/c{i}_values"], out[f"{key}/c{i}_map"] = np.asarray(r[0]), np.asarray(r[1])
                keys = np.asarray(s.key_array())
                b = bits(keys).copy()
                if s.nan_count:
                    b[s.nan_index] = 0
                out[f"{key}/keys"] = b
                out[f"{key}/offsets"] = np.array(s.offsets(), np.int64)
                out[f"{key}/nan"] = np.array([s.nan_count, s.nan_index if s.nan_count else 0], np.int64)
                out[f"{key}/null"] = np.array([s.null_count, s.null_index if s.null_count else 0], np.int64)
                out[f"{key}/query"] = q
                out[f"{key}/query_ordinals"] = np.asarray(s.map_ordinal(q))
                out[f"{key}/query_isin"] = np.asarray(s.isin(q))
    for name, ka, kb in (("merge_nan_left", [1.0, np.nan], [5.0]), ("merge_nan_right", [1.0], [7.0, np.nan])):
        a, b = R.ordered_set("float64", 1), R.ordered_set("float64", 1)
        a.update(np.array(ka))
        b.update(np.array(kb))
        a.merge([b])
        q = np.array(sorted(set(ka + kb) - {np.nan}) + [np.nan])
        out[f"{name}/dtype"], out[f"{name}/nmaps"] = np.array("float64"), np.array(1)
        out[f"{name}/query"], out[f"{name}/query_ordinals"] = q, np.asarray(a.map_ordinal(q)).astype(np.int64)
        out[f"{name}/nan"] = np.array([a.nan_count, a.nan_index], np.int64)
    return out


if __name__ == "__main__":
    data = cases()
    np.savez_compressed(os.path.join(HERE, "set_edges_golden.npz"), **data)
    print("wrote", len(data), "arrays")
