"""The part geometry of csrc/ringcount.cu: interleaved parts (part = cell of the outermost key mod 32 or 64) whenever
ceil(outer cells / parts) rows of the grid fit one part, contiguous ranges of the index otherwise.

Every case is bit-exact against the oracle, conserves the rows, and proves which mapping ran: the last template argument of
k_ring_partition is true for interleaved parts.  The distributions stress both mappings: keys sorted by the outer key (every
warp fills one ring: overflow into direct REDs), an all-NaN outer column (every row in one part), ragged row counts, outer bin
counts that are no multiple of the part count.
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]

from helpers import B200Binby, same_bits  # noqa: E402

pytestmark = pytest.mark.gpu


def launched(fn):
    """the names of the CUDA kernels fn() launched; a profiler session now and then comes back without its kernel records, so `fn`
    is run again when that happens"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = sorted({e.name for e in prof.events() if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset"))})
        if names:
            return names
    raise AssertionError("torch.profiler recorded no CUDA kernel")


N = (1 << 22) + 4097

# name: (key dtype, bins per key (first key fastest), expected parts per lane, interleaved?)
CASES = {
    "2d_f32_1027sq": ("f4", (1024, 1024), 1, True),          # 33 x 1027 = 33,891 cells per part
    "2d_f64_1027sq": ("f8", (1024, 1024), 1, True),
    "2d_f32_outer_not_multiple": ("f4", (1024, 500), 1, True),  # 503 outer cells: parts of 16 and 15 grid rows
    "1d_f32_3M_cells": ("f4", (3_000_000,), 2, True),        # 3,000,003 cells -> 64 interleaved parts of 46,876 cells
    "3d_f32_123cube": ("f4", (120, 120, 120), 2, True),      # 2 x 123^2 = 30,258 cells per part at 64 parts, > 49,151 at 32
    "3d_f64_123cube": ("f8", (120, 120, 120), 2, True),
    "2d_f32_contiguous": ("f4", (50_000, 20), 1, False),     # a grid row of 50,003 cells does not fit a part
    "2d_f64_contiguous": ("f8", (50_000, 20), 1, False),
    "2d_f32_sorted_outer": ("f4", (1024, 1024), 1, True),
    "2d_f32_all_nan_outer": ("f4", (1024, 1024), 1, True),
    "2d_f64_ragged": ("f8", (700, 900), 1, True),
}


def keys_for(case, dt, bins, rng):
    n = N + 2 * 12_347 + 1 if case.endswith("ragged") else N
    keys = [rng.normal(0, 1, n).astype(dt) for _ in bins]
    if case.startswith("1d"):
        keys[0] = rng.uniform(-3.2, 3.2, n).astype(dt)
    if case.startswith("3d"):
        keys = [rng.uniform(-1.1, 1.1, n).astype(dt) for _ in bins]
    for k in keys:
        k[::9973] = np.nan
    if case.endswith("sorted_outer"):
        keys[-1] = np.sort(keys[-1])
    if case.endswith("all_nan_outer"):
        keys[-1][:] = np.nan
    return n, keys


def problem(case, O):
    dt, bins, _, _ = CASES[case]
    rng = np.random.default_rng(1000 + sorted(CASES).index(case))
    n, keys = keys_for(case, dt, bins, rng)
    limits = (-3, 3) if not case.startswith("3d") else (-1, 1)
    return n, [O.scalar(k, *limits, b) for k, b in zip(keys, bins)], [O.agg("count")]


@pytest.fixture(scope="module")
def kernels(tmp_path_factory):
    """the kernels every case launched, recorded with torch.profiler in a fresh process: late in a long pytest process the
    profiler's sessions come back without kernel records more and more often"""
    out = tmp_path_factory.mktemp("prof") / "kernels.json"
    subprocess.check_call([sys.executable, os.path.abspath(__file__), str(out)], cwd=os.path.dirname(HERE))
    return json.loads(out.read_text())


@pytest.mark.parametrize("case", sorted(CASES))
def test_ring_geometry(case, oracle, kernels):
    dt, bins, ppl, interleaved = CASES[case]
    n, binners, aggs = problem(case, oracle)
    got = B200Binby(binners, aggs).run(n, None, "resident")
    names = kernels[case]
    T = "float" if dt == "f4" else "double"
    pattern = rf"k_ring_partition<{T}, {len(bins)}, {ppl}, \d+, (true|false), {'true' if interleaved else 'false'}>"
    assert any(re.search(pattern, s) for s in names), (pattern, sorted(names))
    assert any("k_ring_count" in s for s in names), sorted(names)
    assert int(got[0].sum()) == n
    assert same_bits(oracle.binby(binners, aggs, n)[0], got[0])


if __name__ == "__main__":  # the profiling half of test_ring_geometry, in a process of its own
    from oracle import oracle as O
    O.lib()
    recorded = {}
    for case in sorted(CASES):
        n, binners, aggs = problem(case, O)
        recorded[case] = launched(lambda: B200Binby(binners, aggs).run(n, None, "resident"))
    with open(sys.argv[1], "w") as f:
        json.dump(recorded, f)
