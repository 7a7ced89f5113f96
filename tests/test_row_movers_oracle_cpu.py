"""The fast references of test_gpu_row_movers_edges.py without a GPU: row_movers_oracle.argsort against sort_oracle.argsort and
pa.compute.sort_indices, row_movers_oracle.agg_list against oracle.agg_list."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]
import row_movers_oracle as R  # noqa: E402
import sort_oracle as S  # noqa: E402


@pytest.mark.parametrize("seed", range(6))
def test_string_keys_sort_as_sort_oracle(seed):
    rng = np.random.default_rng(seed)
    kinds = S.NUMERIC + S.TIMES + ["string"]
    for trial in range(20):
        n = int(rng.integers(1, 300))
        keys = []
        for _ in range(rng.integers(1, 5)):
            kind, masked, descending = rng.choice(kinds), rng.random() < 0.4, rng.random() < 0.5
            keys.append(R.string_key(rng, n, masked, descending) if kind == "string" else S.random_key(rng, kind, n, masked, rng.random() < 0.3, descending))
        plain = [k[:3] for k in keys]
        want = S.argsort(plain)
        assert np.array_equal(R.argsort(keys), want)
        assert np.array_equal(S.arrow_argsort(plain), want)


def test_arrow_strings():
    rng = np.random.default_rng(9)
    key = R.string_key(rng, 500, True, False)
    values, mask, _, _ = key
    assert R.arrow_strings(key).to_pylist() == [None if m else v for v, m in zip(values, mask)]


CALLS = [(0, 1), (1, 4), (4, 1027), (1027, 2052), (2052, 4100), (4100, 4101)]


@pytest.mark.parametrize("dtype", S.NUMERIC + [">f8", ">i4"])
@pytest.mark.parametrize("masked", [False, True])
def test_agg_list_matches_oracle(dtype, masked):
    from oracle import oracle as O
    rng = np.random.default_rng(len(dtype) + masked)
    n, ncells = CALLS[-1][1], 7
    cells = rng.integers(0, ncells, n)
    dt = np.dtype(dtype)
    if dt.kind == "b":
        values = rng.random(n) < 0.5
    else:
        values = rng.integers(0, 256, n * dt.itemsize, dtype=np.uint8).view(dt)
        if dt.kind == "f":
            values[rng.random(n) < 0.2] = np.nan
    valid = (rng.random(n) > 0.3).astype(np.uint8) if masked else None
    for dropnan in (False, True):
        for dropnull in (False, True):
            off, vals, nulls = R.agg_list(cells, values, valid, ncells, dropnan, dropnull, CALLS)
            want_off, want, _, _ = O.agg_list(cells, values, valid, ncells, dropnan, dropnull, calls=CALLS)
            assert np.array_equal(off, want_off)
            assert vals.dtype == want.dtype
            isz = vals.dtype.itemsize
            assert np.array_equal(vals.view(f"u{isz}")[~nulls], want.view(f"u{isz}")[~nulls])
            assert nulls.sum() == (0 if dropnull or not masked else np.count_nonzero(valid[R.call_starts(n, CALLS) + (np.arange(n) - R.call_starts(n, CALLS)) % 1024] == 0))
