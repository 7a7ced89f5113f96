"""The reference's sort tests (tests/sort_test.py) as data: each case is the frame's columns, its filter, the sort's arguments and
the expected columns of the result.  test_sort's frame is `arange(10)` in a shuffled order (the reference shuffles with
`sample(frac=1, random_state=42)`; any order that is not sorted tests the same thing)."""
import numpy as np

SHUFFLED = np.array([7, 1, 5, 2, 9, 0, 3, 8, 4, 6])
X10 = list(range(10))

MULTI = {"x": np.array([5, 3, 1, 1, 5]), "y": np.array([0, 3, 4, 2, 1]), "z": np.array(["dog", "cat", "cat", "dog", "mouse"], dtype=object)}

CASES = {
    # test_sort
    "x": ({"x": SHUFFLED}, None, dict(by="x"), {"x": X10}),
    "-x": ({"x": SHUFFLED}, None, dict(by="-x"), {"x": X10[::-1]}),
    "-x descending": ({"x": SHUFFLED}, None, dict(by="-x", ascending=False), {"x": X10}),
    "x descending": ({"x": SHUFFLED}, None, dict(by="x", ascending=False), {"x": X10[::-1]}),
    # test_sort_filtered
    "filtered": ({"x": np.array([2, 3, 1, 5, 7, 6])}, "x > 4", dict(by="x"), {"x": [5, 6, 7]}),
    # test_sort_multikey
    "numeric keys": (MULTI, None, dict(by=["x", "y"]), {"x": [1, 1, 3, 5, 5], "y": [2, 4, 3, 0, 1], "z": ["dog", "cat", "cat", "dog", "mouse"]}),
    "string key first": (MULTI, None, dict(by=["z", "x"]), {"x": [1, 3, 1, 5, 5], "y": [4, 3, 2, 0, 1], "z": ["cat", "cat", "dog", "dog", "mouse"]}),
    "mixed order": (MULTI, None, dict(by=["z", "x"], ascending=[False, True]),
                    {"x": [5, 1, 5, 1, 3], "y": [1, 2, 0, 4, 3], "z": ["mouse", "dog", "dog", "cat", "cat"]}),
    # test_sort_strings_masked
    "strings ascending": ({"x": np.array(["Groningen", "Skopje", None, "Amsterdam", "Ohrid"], dtype=object)}, None, dict(by="x"),
                          {"x": ["Amsterdam", "Groningen", "Ohrid", "Skopje", None]}),
    "strings descending": ({"x": np.array(["Groningen", "Skopje", None, "Amsterdam", "Ohrid"], dtype=object)}, None, dict(by="x", ascending=False),
                           {"x": ["Skopje", "Ohrid", "Groningen", "Amsterdam", None]}),
    # test_sort_empty
    "empty": ({"x": np.array([5, 1, 4]), "y": np.array([1, 2, 3])}, "y > 10", dict(by="x"), {"x": [], "y": []}),
}
