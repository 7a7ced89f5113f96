"""The join restatement (join_oracle.py) against the reference's join tests (join_cases.py) and the differences DESIGN.md section 3
names; no GPU needed."""
import math

import numpy as np
import pytest

import join_cases
import join_oracle as J


def frame(spec):
    columns, filter = spec
    return J.OFrame(columns, join_cases.filter_mask(columns, filter))


def same(a, b):
    return len(a) == len(b) and all(x == y or (isinstance(x, float) and isinstance(y, float) and math.isnan(x) and math.isnan(y)) for x, y in zip(a, b))


def check(result, expected):
    for name, want in expected.items():
        if name == "__names__":
            assert set(result.columns) == want
            continue
        assert same(result.values(name), want), (name, result.values(name), want)


@pytest.mark.parametrize("case", join_cases.CASES, ids=[c[0] for c in join_cases.CASES])
def test_reference_case(case):
    _, left, right, kwargs, expected = case
    check(J.join(frame(left), frame(right), **kwargs), expected)


@pytest.mark.parametrize("case", join_cases.ERRORS, ids=[c[0] for c in join_cases.ERRORS])
def test_reference_error(case):
    _, left, right, kwargs, exc, text = case
    with pytest.raises(exc, match=text):
        J.join(frame(left), frame(right), **kwargs)


def test_filtered_left_keeps_unfiltered_rows():
    """test_left_a_b_filtered: the filter stays, every row was matched"""
    left = frame((join_cases.df_a(), "x > 0"))
    out = J.join(left, frame((join_cases.df_b(), None)), left_on="a", right_on="b", rsuffix="_r")
    assert out.values("x_r", filtered=False) == [2, 1, None]


def test_duplicates_order_by_left_then_right_row():
    """difference 1: appended rows ordered by (left row, right overflow row)"""
    left = J.OFrame({"k": np.array([5, 7, 5]), "v": np.arange(3)})
    right = J.OFrame({"k": np.array([7, 5, 5, 7, 5]), "w": np.arange(10, 15)})
    out = J.join(left, right, on="k", allow_duplication=True, rsuffix="_r")
    assert out.values("v") == [0, 1, 2, 0, 0, 1, 2, 2]
    assert out.values("w") == [11, 10, 11, 12, 14, 13, 12, 14]


def test_masked_left_key_with_duplicates():
    """difference 3: a masked left key maps to the right's null row and adds no pairs"""
    left = J.OFrame({"k": np.ma.array([1, 2, 3], mask=[False, True, False])})
    right = J.OFrame({"k": np.ma.array([1, 1, 0], mask=[False, False, True]), "w": np.array([10, 11, 12])})
    out = J.join(left, right, on="k", allow_duplication=True, rsuffix="_r")
    assert out.values("w") == [10, 12, None, 11]


def test_filtered_left_duplicates_take_unfiltered_rows():
    """difference 4: the repeated rows are the left's unfiltered rows, and keep their filter value"""
    left = J.OFrame({"k": np.array([1, 2, 1]), "v": np.array([0, 1, 2])}, filter=np.array([False, True, True]))
    right = J.OFrame({"k": np.array([1, 1]), "w": np.array([10, 11])})
    out = J.join(left, right, on="k", allow_duplication=True, rsuffix="_r")
    assert out.values("v", filtered=False) == [0, 1, 2, 0, 2]
    assert out.values("w", filtered=False) == [10, None, 10, 11, 11]
    assert out.values("v") == [1, 2, 2]


def test_numpy_join_matches_restatement():
    rng = np.random.default_rng(3)
    lk, rk = rng.integers(0, 50, 300), rng.integers(0, 40, 120)
    out = J.join(J.OFrame({"k": lk, "v": np.arange(300)}), J.OFrame({"k": rk, "w": np.arange(120)}), on="k", allow_duplication=True, rsuffix="_r")
    lrows, rrows = J.numpy_join(lk, rk)
    assert out.values("v") == lrows.tolist()
    assert out.values("w") == [None if r < 0 else int(r) for r in rrows]
