"""Generate tests/golden/edges_golden.npz from the COMPILED, UNMODIFIED reference (oracle/_ref).

Run where /root/reference exists and `make -C oracle ref` has been run:

    python tests/golden/make_golden_edges.py

Same case layout as binstats_golden.npz (make_golden.add_case).  Two groups:
  * single-cell known answers where the device's rule is documented in DESIGN §3 (integer sum_moment out of range and past
    2^53, min / max over both signed zeros), integer sums that wrap modulo 2^64, exact integer powers for moments 5..8;
  * a fixed set of edge-value problems drawn by tests/helpers.py random_case(edges=True).
The archive is written with fixed zip timestamps, so a rerun reproduces it byte for byte.
"""
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import oracle as O  # noqa: E402
from helpers import random_case  # noqa: E402
from make_golden import add_case  # noqa: E402


def one_cell(values):
    """a scalar binner that puts every row into cell 2 (the first in-range cell)"""
    return [O.scalar(np.full(len(values), 0.5), 0, 1, 1)]


def cases():
    out = {}
    i8, u8 = np.iinfo(np.int64), np.iinfo(np.uint64)
    v = np.array([3_000_000], "i8")
    add_case(out, "kat_moment3_int64_out_of_range", one_cell(v), [O.agg("sum_moment", v, moment=3)], 1)
    v = np.array([3_000_000], "u8")
    add_case(out, "kat_moment3_uint64_out_of_range", one_cell(v), [O.agg("sum_moment", v, moment=3)], 1)
    v = np.array([30000, 30001, 29999, 1], "i8")
    add_case(out, "kat_moment4_past_2p53", one_cell(v), [O.agg("sum_moment", v, moment=4)], 4)
    v = np.array([0.0, -0.0])
    add_case(out, "kat_minmax_signed_zeros", one_cell(v), [O.agg("min", v), O.agg("max", v)], 2)
    v = np.array([i8.max, i8.max, 1, i8.min, -1, i8.max], "i8")
    add_case(out, "kat_sum_wraps_int64", one_cell(v), [O.agg("sum", v)], len(v))
    v = np.array([u8.max, 5, 1 << 63, 1 << 63, u8.max - 1], "u8")
    add_case(out, "kat_sum_wraps_uint64", one_cell(v), [O.agg("sum", v)], len(v))
    v = np.array([3, 7, 11, 13, -5, 1, 0, -1], "i8")  # every power below 2^53: exact
    add_case(out, "kat_moments_5_to_8_exact", one_cell(v), [O.agg("sum_moment", v, moment=m) for m in (5, 6, 7, 8)], len(v))
    for seed in range(16):
        rng = np.random.default_rng(9100 + seed)
        n = int(rng.integers(1, 1200))
        binners, aggs = random_case(rng, n, edges=True)
        add_case(out, f"edges_{seed:02d}", binners, aggs, n)
    return out


def save(path, arrays):
    """np.savez_compressed with fixed zip timestamps (reproducible bytes)"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(info, "w") as f:
                np.lib.format.write_array(f, np.asanyarray(arrays[name]), allow_pickle=False)


if __name__ == "__main__":
    path = os.path.join(HERE, "edges_golden.npz")
    data = cases()
    save(path, data)
    print("wrote", len(data), "arrays,", os.path.getsize(path) // 1024, "KiB")
