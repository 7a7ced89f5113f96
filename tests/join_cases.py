"""The reference's join tests (tests/join_test.py) that do not need string keys, as data: the string keys a / b / c / f are rewritten
as integer codes (A=0, B=1, C=2, D=3, X=10, Y=11, Z=12, missing = masked) with the same expected values.  Each case is
(name, left, right, join keyword arguments, expected columns or the error it raises); a frame is (columns, filter expression or
None).  Filters are numeric expressions both numpy (`filter_mask`) and the device evaluate."""
import numpy as np


def df_a():
    return {"a": np.array([0, 1, 2]), "x": np.array([0., 1., 2.]), "y": np.ma.array([0., 9., 2.], mask=[False, True, False]),
            "m": np.ma.array([1, 2, 3], mask=[False, True, False])}


def df_b():
    return {"b": np.array([0, 1, 3]), "x": np.array([2., 1., 0.]), "y": np.ma.array([9., 1., 2.], mask=[True, False, False]),
            "m": np.ma.array([3, 1, 2], mask=[True, False, False])}


def df_dup():
    return {"b": np.array([0, 1, 0]), "x": np.array([2., 1., 2.]), "y": np.ma.array([9., 1., 9.], mask=[True, False, False]),
            "m": np.ma.array([3, 1, 2], mask=[True, True, False])}


def df_c():
    return {"c": np.array([1, 2]), "z1": np.array([-1., -2.]), "z2": np.array([True, False])}


def df_d():
    return {"a": np.array([1, 2, 3]), "x1": np.array(["dog", "cat", "mouse"], dtype=object), "x2": np.array([3.1, 25, np.nan])}


def df_e():
    return {"a": np.array([10, 11, 12]), "x1": np.array(["dog", "cat", "mouse"], dtype=object), "x2": np.array([3.1, 25, np.nan])}


def df_f():
    return {"f": np.ma.array([1, 2, 0], mask=[False, False, True]), "w1": np.array(["dog", "cat", "mouse"], dtype=object),
            "w2": np.array([True, False, True])}


def df_dt1():
    return {"date": np.array(['2009-10-12T03:00:00', '2009-10-12T11:00:00', '2009-10-12T12:00:00', '2009-12-12T03:00:00'], dtype="datetime64[ns]"),
            "value": np.array([1, 2, 3, 4])}


def df_dt2():
    return {"date": np.array(['2009-10-12T03:00:00', '2009-10-12T11:00:00', '2009-12-12T03:00:00'], dtype="datetime64[ns]"),
            "value": np.array([11, 22, 44])}


def filter_mask(columns, expression):
    """a numeric filter expression over `columns`, in numpy"""
    if expression is None:
        return None
    env = {k: np.ma.getdata(v) for k, v in columns.items()}
    return np.asarray(eval(expression, {"__builtins__": {}}, env), bool)


CASES = [
    ("join_masked", (df_a(), None), (df_b(), None), dict(left_on="m", right_on="m", rsuffix="_r"),
     {"m": [1, None, 3], "m_r": [1, None, None]}),
    ("join_nomatch", (df_a(), None), (df_e(), None), dict(on="a", rprefix="r_"), {"x2": [None, None, None]}),
    ("left_a_b", (df_a(), None), (df_b(), None), dict(left_on="a", right_on="b", rsuffix="_r"),
     {"a": [0, 1, 2], "b": [0, 1, None], "x": [0, 1, 2], "x_r": [2, 1, None], "y": [0, None, 2], "y_r": [None, 1, None]}),
    ("left_a_b_filtered", (df_a(), "x > 0"), (df_b(), None), dict(left_on="a", right_on="b", rsuffix="_r"),
     {"a": [1, 2], "b": [1, None], "x": [1, 2], "x_r": [1, None], "y": [None, 2], "y_r": [1, None]}),
    # the reference's filter is b.str.contains('A|B'): rows A and B, i.e. codes 0 and 1
    ("left_a_b_filtered_right", (df_a(), None), (df_b(), "b < 2"), dict(how="left", on="x", rsuffix="_r"),
     {"x": [0, 1, 2], "a": [0, 1, 2], "y": [0, None, 2], "m": [1, None, 3], "b": [None, 1, 0], "x_r": [None, 1, 2], "y_r": [None, 1, None],
      "m_r": [None, 1, None]}),
    ("right_x_x", (df_a(), None), (df_b(), None), dict(on="x", rsuffix="_r", how="right"),
     {"a": [2, 1, 0], "b": [0, 1, 3], "x": [2, 1, 0], "x_r": [2, 1, 0], "y": [2, None, 0], "y_r": [None, 1, 2]}),
    ("left_a_c", (df_a(), None), (df_c(), None), dict(left_on="a", right_on="c", how="left"),
     {"a": [0, 1, 2], "x": [0, 1, 2], "y": [0., None, 2.], "m": [1, None, 3], "c": [None, 1, 2], "z1": [None, -1., -2.], "z2": [None, True, False]}),
    ("left_dup", (df_a(), None), (df_dup(), None), dict(left_on="a", right_on="b", rsuffix="_r", allow_duplication=True),
     {"a": [0, 1, 2, 0], "b": [0, 1, None, 0], "x": [0, 1, 2, 0], "x_r": [2, 1, None, 2], "y": [0, None, 2, 0], "y_r": [None, 1, None, 9],
      "m": [1, None, 3, 1], "m_r": [None, None, None, 2]}),
    ("inner_a_b", (df_a(), None), (df_b(), None), dict(left_on="a", right_on="b", rsuffix="_r", how="inner"),
     {"a": [0, 1], "b": [0, 1], "x": [0, 1], "x_r": [2, 1], "y": [0, None], "y_r": [None, 1]}),
    ("inner_a_d", (df_a(), None), (df_d(), None), dict(on="a", right_on="a", how="inner", rsuffix="_r"),
     {"a": [1, 2], "x": [1, 2], "y": [None, 2], "m": [None, 3], "x1": ["dog", "cat"], "x2": [3.1, 25.]}),
    ("join_filtered_inner", (df_a(), "x > 0"), (df_b(), None), dict(on="x", how="inner", rsuffix="_", allow_duplication=True),
     {"x": [1., 2.], "a": [1, 2], "b": [1, 0]}),
    ("join_duplicate_column", (df_a(), None), (df_a(), None), dict(on="a", lsuffix="_left", rsuffix="_right"),
     {"__names__": {"a_left", "x_left", "y_left", "m_left", "a_right", "x_right", "y_right", "m_right"}, "x_right": [0, 1, 2]}),
    ("join_no_right_columns_left", ({"a": np.array([1, 2, 3])}, None), ({"a": np.array([1, 10])}, None), dict(on="a", how="inner"),
     {"a": [1]}),
    ("join_on_nan_primitive", ({"id": np.array([0., 1., np.nan]), "x": np.array([1, 2, 3])}, None),
     ({"id": np.array([0., 1., 2.]), "y": np.array([2, 3, 4])}, None), dict(on="id"), {"x": [1, 2, 3], "y": [2, 3, None]}),
    ("join_on_null_primitive", ({"id": np.ma.array([0., 1., 0.], mask=[False, False, True]), "x": np.array([1, 2, 3])}, None),
     ({"id": np.array([0., 1., 2.]), "y": np.array([2, 3, 4])}, None), dict(on="id"), {"x": [1, 2, 3], "y": [2, 3, None]}),
    ("with_masked_no_short_circuit", ({"id": np.array([0, 1, 2]), "x": np.array([1, 2, 3])}, None),
     ({"id": np.array([0, 1, 2]), "y": np.ma.array([2, 3, 4], mask=[False, True, False])}, None), dict(on="id"), {"y": [2, None, 4]}),
    ("join_datetime", (df_dt1(), None), (df_dt2(), None), dict(on="date", rsuffix="_right"),
     {"value": [1, 2, 3, 4], "value_right": [11, 22, None, 44]}),
    ("join_on_masked_key", (df_a(), None), (df_f(), None), dict(left_on="a", right_on="f"),
     {"a": [0, 1, 2], "w1": [None, "dog", "cat"], "w2": [None, True, False]}),
    ("no_on", (df_a(), None), (df_b(), None), dict(rsuffix="_r"), {"b": [0, 1, 3], "x_r": [2, 1, 0]}),
]

# (name, left, right, kwargs, the exception and a piece of its message)
ERRORS = [
    ("collision", (df_a(), None), (df_b(), None), dict(left_on="a", right_on="b"), ValueError, "collision"),
    ("duplication", (df_a(), None), (df_dup(), None), dict(left_on="a", right_on="b", rsuffix="_r"), ValueError, "duplication"),
    ("how", (df_a(), None), (df_b(), None), dict(left_on="a", right_on="b", rsuffix="_r", how="outer"), ValueError, "not supported"),
]

