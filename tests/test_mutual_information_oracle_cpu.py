"""The numpy restatement of df.mutual_information (tests/mutual_information_oracle.py) against the committed golden vectors (the
reference's own method over the compiled superagg and vaexfast), and against the reference's method itself where its sources are
present."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import mutual_information_oracle as MO  # noqa: E402
from helpers import same_bits  # noqa: E402

REFERENCE_VAEX = "/root/reference/packages/vaex-core/vaex"
have_reference = pytest.mark.skipif(not os.access(os.path.join(REFERENCE_VAEX, "dataframe.py"), os.R_OK),
                                    reason="the reference sources are not on this machine")


def frame_columns(frames, case):
    columns = frames[case["frame"]]
    if case["filter"]:
        keep = np.asarray(columns[case["filter"]], bool)
        columns = {k: v[keep] for k, v in columns.items()}
    return columns


def run(columns, kwargs):
    with np.errstate(all="ignore"):
        return MO.mutual_information(columns, **kwargs)


def test_golden_against_restatement():
    frames, cases = MO.load_golden()
    assert len(cases) >= 40
    for name, case in cases.items():
        columns = frame_columns(frames, case)
        if "error" in case:
            with pytest.raises(Exception) as info:
                run(columns, case["kwargs"])
            assert type(info.value).__name__ == case["error"], name
            continue
        got = run(columns, case["kwargs"])
        assert type(got).__name__ == case["result_type"], name
        if isinstance(got, tuple):
            got, labels = got
            assert [list(v) if isinstance(v, tuple) else v for v in labels] == case["labels"], name
        assert got.shape == case["result"].shape, name
        assert same_bits(np.asarray(got), case["result"]), name


def test_golden_known_answers():
    _, cases = MO.load_golden()
    np.testing.assert_array_almost_equal(cases["df_local_known"]["result"], 2.043192)  # reference tests/agg_test.py:447
    assert cases["df_local_known"]["result"].shape == ()  # one pair: a 0-d ndarray, not a scalar
    assert cases["df_local_binby1"]["result"].shape == (2,)
    assert cases["df_local_binby2"]["result"].shape == (2, 3)
    assert cases["df_local_binby3"]["result"].shape == (2, 3, 4)
    assert cases["matrix_dim3"]["result"].shape == (2, 2, 2)
    assert cases["list_vs_list"]["result"].shape == (3, 2)
    assert np.all(cases["ab_dimension1"]["result"] == 0.0) and cases["all_empty"]["result"] == 0.0
    # the sorted, deduplicated combinations get the limits: (b, a) and (a, b) with per-axis limits give the same answer
    assert same_bits(cases["mi_limits_sorted"]["result"][:1], cases["mi_limits_pair_per_axis"]["result"].reshape(1))
    assert cases["sort_single_pair"]["labels"] == ["a"]  # x[k] of the string "ab"
    assert cases["sort_matrix_index_error"]["error"] == "IndexError"
    assert cases["sort_binby_raises"]["error"] == "TypeError"
    assert cases["binby_dim4"]["error"] == "ValueError"
    assert cases["string_x_list_y"]["error"] == "TypeError"


def test_reshape_not_transpose_with_binby_and_several_combinations():
    """(ncomb, *binby) values reshaped to binby_shape + shape_result: element [i, j] is not combination j of binby cell i"""
    frames, cases = MO.load_golden()
    case = cases["pairs_binby1"]
    columns = frame_columns(frames, case)
    per_pair = [MO.mutual_information(columns, x=p, y=q, mi_shape=8, binby=["k"], shape=4) for p, q in (("a", "b"), ("b", "c"), ("a", "c"))]
    stacked = np.array(per_pair)  # (3 pairs, 4 cells) in the caller's order
    assert same_bits(case["result"], stacked.reshape(4, 3))
    assert not same_bits(case["result"], stacked.T)


def test_bound_covers_rounding_on_exact_outer_products():
    """c = a_i * b_j has MI 0 in exact arithmetic; the float64 restatement lands within the stated bound of it"""
    rng = np.random.default_rng(3)
    for shape in [(2, 2), (7, 5), (256, 256), (3, 4, 5)]:
        factors = [rng.integers(1, 1000, n) for n in shape]
        counts = factors[0].astype(np.int64)
        for f in factors[1:]:
            counts = np.multiply.outer(counts, f)
        mi = MO.mi_cell(counts.astype(np.float64))
        assert abs(mi) <= MO.bound(counts), shape


def test_diagonal_is_the_entropy():
    counts = np.diag(np.arange(1, 40, dtype=np.int64))
    p = np.arange(1, 40) / np.arange(1, 40).sum()
    entropy = -np.sum(p * np.log(p))
    assert abs(MO.mi_cell(counts.astype(np.float64)) - entropy) <= MO.bound(counts)


@have_reference
def test_restatement_matches_the_reference_method(ref):
    """random frames through the reference's own method (ast-extracted, over the compiled superagg / vaexfast) and the restatement"""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_mutual_information as G
    method = G.reference_method(REFERENCE_VAEX)
    for seed in range(8):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(50, 2000))
        u = rng.normal(size=n)
        columns = dict(u=u, v=(u + rng.normal(size=n)).astype(np.float32), t=rng.integers(0, 5, n), s=rng.random(n) < 0.5)
        kwargs = [dict(x="u", y="v", mi_shape=int(rng.integers(1, 40))),
                  dict(x=["u", "v", "t"], mi_shape=[5, 9], binby=["t"], shape=3, selection="s"),
                  dict(x=[["v", "u"], ["t", "u"]], dimension=2, mi_shape=6, binby=["u", "v"], shape=[2, 3]),
                  dict(x=["u", "v", "t"], dimension=3, mi_shape=3, sort=seed > 4)][seed % 4]
        try:
            with np.errstate(all="ignore"):
                want = method(G.Stub(columns), **kwargs)
        except Exception as e:  # x[k] past the end of x for the sorted matrix form
            with pytest.raises(type(e)):
                run(columns, kwargs)
            continue
        got = run(columns, kwargs)
        assert type(got) is type(want)
        if isinstance(want, tuple):
            assert got[1] == want[1]
            got, want = got[0], want[0]
        assert same_bits(np.asarray(got), np.asarray(want)), (seed, kwargs)


@have_reference
def test_golden_regenerates_byte_for_byte(ref, tmp_path):
    out = tmp_path / "mutual_information_golden.npz"
    subprocess.check_call([sys.executable, os.path.join(HERE, "golden", "make_golden_mutual_information.py"), str(out), REFERENCE_VAEX])
    assert out.read_bytes() == open(MO.GOLDEN, "rb").read()
