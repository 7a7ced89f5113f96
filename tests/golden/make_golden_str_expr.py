"""Writes tests/golden/str_expr_golden.npz: the compiled reference's string predicates and measures (oracle/_ref/strfunc_shim, the
unmodified src/superstring.hpp) over the edge corpus of tests/str_expr_oracle.py, for the GPU tests, which run where the reference
is not.  contains and count come from src/strings.cpp, which is not built: their vectors are the restatement's, pinned against
bytes.find / bytes.count by tests/test_str_expr_oracle_cpu.py.

usage:  python tests/golden/make_golden_str_expr.py     (after __graft_entry__.build())"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))
import str_expr_oracle as O  # noqa: E402


def reference(shim, name, pattern, start, end, rows=O.ROWS, nulls=O.NULLS):
    """one call of the compiled reference over `rows`"""
    off, data, mask = O.buffers(rows, nulls)
    if name == "equals2":
        rows2, nulls2 = O.second_column(rows, nulls)
        off2, data2, mask2 = O.buffers(rows2, nulls2)
        return np.asarray(shim.equals2(off, data, mask, off2, data2, mask2))
    if name == "notequals":  # str_notequals = ~str_equals (vaex/functions.py:1015-1060)
        return ~np.asarray(shim.equals(off, data, mask, pattern))
    if name in ("len", "byte_length"):
        return np.asarray(getattr(shim, name)(off, data, mask))
    if name in ("find", "rfind"):
        return np.asarray(shim.find(off, data, mask, pattern, start, end, name == "find"))
    if name in ("contains", "count"):
        return O.evaluate(name, rows, nulls, pattern)
    return np.asarray(getattr(shim, name)(off, data, mask, pattern))


def main():
    import strfunc_shim
    off, data, mask = O.buffers(O.ROWS, O.NULLS)
    rows2, nulls2 = O.second_column()
    off2, data2, mask2 = O.buffers(rows2, nulls2)
    out = dict(offsets=off, bytes=data, nulls=mask, offsets2=off2, bytes2=data2, nulls2=mask2)
    for name, pattern, start, end in O.calls():
        out[O.key(name, pattern, start, end)] = reference(strfunc_shim, name, pattern, start, end)
    path = os.path.join(HERE, "str_expr_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out) - 6} result vectors over {len(O.ROWS)} rows")


if __name__ == "__main__":
    main()
