"""The numpy restatement of percentile_approx's finish (tests/percentile_oracle.py) against the compiled, unmodified
vaexfast.grid_find_edges, and the committed golden vectors (the reference's own finish) against the restatement."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import percentile_oracle as PO  # noqa: E402
from helpers import same_bits  # noqa: E402

REFERENCE_DATAFRAME = "/root/reference/packages/vaex-core/vaex/dataframe.py"


def random_cumulative(rng, lead, plen):
    """non-decreasing int64 rows: ties (zero counts), empty rows and totals up to 2^62"""
    scale = rng.choice([3, 1000, 2**40, 2**55])
    counts = rng.integers(0, scale, lead + (plen,), dtype=np.int64)
    counts[rng.random(counts.shape) < 0.4] = 0
    if lead:
        counts.reshape(-1, plen)[rng.random(int(np.prod(lead))) < 0.2] = 0
    cum = np.cumsum(counts, -1)
    assert cum.max(initial=0) <= 2**62
    return cum


def random_targets(rng, cum):
    total = cum[..., -1]
    t = np.floor(rng.random(total.shape) * (total + 2).astype(np.float64))
    pick = rng.random(total.shape)
    t = np.where(pick < 0.15, 0.0, t)  # target 0
    t = np.where((pick >= 0.15) & (pick < 0.3), total.astype(np.float64) + 1, t)  # beyond the total
    t = np.where((pick >= 0.3) & (pick < 0.4), total.astype(np.float64), t)  # exactly the total
    return np.array(t, np.float64)


@pytest.mark.parametrize("lead", [0, 1])
@pytest.mark.parametrize("seed", range(12))
def test_edges_match_compiled_grid_find_edges(ref, lead, seed):
    rng = np.random.default_rng(seed * 7 + lead)
    shape = tuple(int(n) for n in rng.integers(1, 40, lead))
    cum = random_cumulative(rng, shape, int(rng.choice([1, 2, 3, 17, 300])))
    t = random_targets(rng, cum)
    for got, want in zip(PO.edges_numpy(cum, t), PO.edges_vaexfast(cum, t)):
        assert same_bits(np.asarray(got, np.int64), np.asarray(want, np.int64))


@pytest.mark.parametrize("lead", [0, 1])
@pytest.mark.parametrize("seed", range(12))
def test_finish_matches_compiled_search(ref, lead, seed):
    """the whole finish with either search, int and float percentages, float32 / int64 / Python limits"""
    rng = np.random.default_rng(500 + seed * 7 + lead)
    P = int(rng.choice([1, 2, 16, 257]))
    shape = tuple(int(n) + 3 for n in rng.integers(1, 20, lead)) + (P + 3,)
    counts = rng.integers(0, int(rng.choice([4, 2**50])), shape, dtype=np.int64)
    counts[rng.random(shape) < 0.5] = 0
    limit = [np.array([-1.5, 2.25], np.float32), np.array([-3, 1000], np.int64), [-4.0, 4.0]][seed % 3]
    pct = [[7, 50, 93], [12.5, 50.0], 50, 66.6][seed % 4]
    with np.errstate(all="ignore"):
        got = PO.finish_one(counts, limit, pct, edges="numpy")
        want = PO.finish_one(counts, limit, pct, edges="vaexfast")
    assert type(got) is type(want) and same_bits(np.asarray(got), np.asarray(want))


@pytest.mark.parametrize("lead", [2, 3])
@pytest.mark.parametrize("seed", range(6))
def test_deviation_per_cell_for_two_or_more_binby_dimensions(ref, lead, seed):
    """with two or more binby dimensions the restatement gives every cell what the compiled search gives that cell's row of the grid
    reshaped to (cells, P + 2): the reference's one-dimensional answer, not its multi-dimensional search, which reads outside the grid"""
    rng = np.random.default_rng(900 + seed * 7 + lead)
    shape = tuple(int(n) for n in rng.integers(1, 9, lead))
    cum = random_cumulative(rng, shape, int(rng.choice([1, 5, 64])))
    t = random_targets(rng, cum)
    left, right = PO.edges_numpy(cum, t)
    flat = cum.reshape(-1, cum.shape[-1])
    want_left, want_right = PO.edges_vaexfast(flat, t.reshape(-1))
    assert same_bits(left.reshape(-1), want_left) and same_bits(right.reshape(-1), want_right)


def test_golden_against_restatement():
    cases = PO.load_golden()
    assert len(cases) >= 25
    for name, c in cases.items():
        with np.errstate(all="ignore"):
            got = PO.finish_one(c["counts"], c["limit"], c["percentage"])
        assert type(got).__name__ == c["result_type"], name
        assert same_bits(np.asarray(got), c["result"]), name


def test_golden_integral_and_float_percentages_differ_past_2_53():
    cases = PO.load_golden()
    assert not same_bits(cases["binby1_big_int"]["result"], cases["binby1_big_float"]["result"])
    assert not same_bits(cases["nobinby_big_int"]["result"], cases["nobinby_big_float"]["result"])


def test_binby_with_0_or_100_mixed_in_is_numpys_inhomogeneous_shape_error():
    counts = np.ones((7, 12), np.int64)
    with pytest.raises(ValueError, match="inhomogeneous"):
        PO.finish_one(counts, [0.0, 1.0], [0, 50])


@pytest.mark.skipif(not os.access(REFERENCE_DATAFRAME, os.R_OK), reason="the reference sources are not on this machine")
def test_golden_regenerates_byte_for_byte(ref, tmp_path):
    out = tmp_path / "percentile_golden.npz"
    subprocess.check_call([sys.executable, os.path.join(HERE, "golden", "make_golden_percentile.py"), str(out), REFERENCE_DATAFRAME])
    assert out.read_bytes() == open(PO.GOLDEN, "rb").read()
