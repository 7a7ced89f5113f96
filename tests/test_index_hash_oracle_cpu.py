"""The numpy restatement of index_hash<T> (tests/index_hash_oracle.py) against the committed golden vectors (the compiled reference's
own classes) and against the compiled classes themselves where oracle/_ref exists: bit for bit where the reference is sequential
(one update at start_index 0; increasing start_index without NaN / null; merges in row order), and the stated deviations elsewhere."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import index_hash_oracle as IO  # noqa: E402
import make_golden_index_hash as G  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "index_hash_golden.npz")


def assert_same(got, want, name):
    assert set(got) == set(want), name
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), f"{name}: {k}"


def test_golden_against_restatement():
    golden = G.load(GOLDEN)
    assert len(golden) == 99
    for name, (case, res) in golden.items():
        assert_same(G.run(IO.classes, case), res, name)


def test_golden_covers_the_conditions():
    golden = G.load(GOLDEN)
    assert {c["dtype"] for c, _ in golden.values()} == set(G.DTYPES)
    assert {c["nmaps"] for c, _ in golden.values()} == {1, 3, 7}
    assert any(c["merges"] for c, _ in golden.values())
    assert any(len(c["updates"]) > 1 for c, _ in golden.values())
    assert any(r["scalars"][3] for _, r in golden.values())  # NaN
    assert any(r["scalars"][4] for _, r in golden.values())  # null
    assert any(r["scalars"][2] for _, r in golden.values())  # duplicates


def test_restatement_against_compiled_reference(ref):
    su = ref.modules()[1]
    for name, case in G.cases().items():
        assert_same(G.run(IO.classes, case), G.run(lambda dt: getattr(su, "index_hash_" + dt), case), name)


def test_issue_example():
    h = IO.RefAPI("int64")
    h.update(np.array([5, 7, 5, 9, 7, 5]), 0)
    h.update(np.array([7, 11, 5]), 6)
    assert (len(h), h.count) == (9, 4)
    rows, unknown = IO.IndexHash.map_index(h, np.array([5, 7, 9, 11, 3]))
    assert rows.tolist() == [0, 1, 3, 7, -1] and unknown
    left, right = h.map_index_duplicates(np.array([3, 7, 5, 9]), 100)
    assert left.tolist() == [101, 101, 102, 102, 102] and right.tolist() == [4, 6, 2, 5, 8]


def test_map_index_foreign_dtype_and_forcecast(ref):
    su = ref.modules()[1]
    h = su.index_hash_int64(1)
    h.update(np.array([5.9, 7.2, 5.1]))  # update force-casts
    assert h.has_duplicates and h.map_index(np.array([5, 7], np.int64)).tolist() == [0, 1]
    with pytest.raises(TypeError):
        h.map_index(np.array([5.0]))
    assert h.map_index(np.array([5, 7], np.int32)).tolist() == [0, 1]  # a safe cast is accepted


def test_narrow_out_truncates(ref):
    su = ref.modules()[1]
    h = su.index_hash_int64(1)
    h.update(np.arange(300, dtype=np.int64))
    look = np.array([299, 128, 127, -5])
    for w in G.WIDTHS:
        o = np.zeros(4, w)
        assert h.map_index(look, o)
        assert np.array_equal(o, IO.truncate([299, 128, 127, -1], w))


def test_len_count_with_nan_and_null(ref):
    su = ref.modules()[1]
    keys = np.array([1.0, np.nan, 2.0, np.nan, 1.0, 3.0])
    mask = np.array([0, 0, 0, 0, 0, 1], np.uint8)
    for h in (su.index_hash_float64(1), IO.RefAPI("float64")):
        h.update(keys, mask, 0)
        assert (len(h), h.count, h.nan_count, h.null_count, h.has_duplicates) == (5, 4, 2, 1, True)
        assert h.map_index_masked(np.array([np.nan, 9.0]), np.array([0, 1], np.uint8)).tolist() == [3, 5]
    # only NaN / null repeat: no duplicates
    for h in (su.index_hash_float64(1), IO.RefAPI("float64")):
        h.update(np.array([np.nan, 4.0, np.nan]), np.array([0, 0, 0], np.uint8), 0)
        assert not h.has_duplicates and len(h) == 2


# ---- the deviations: the reference's answer depends on chunk order; the restatement (and the device) give the sequential one ------

def test_deviation_nan_null_row_is_global(ref):
    su = ref.modules()[1]
    a, b = su.index_hash_float64(1), IO.RefAPI("float64")
    for h in (a, b):
        h.update(np.array([1, np.nan, 2, np.nan]), 0)
        h.update(np.array([3, np.nan, 4]), 10)
    assert a.map_index(np.array([np.nan])).tolist() == [1]   # call-local offset of the last call
    assert b.map_index(np.array([np.nan])).tolist() == [11]  # the largest global NaN row


def test_deviation_merge(ref):
    su = ref.modules()[1]
    ra, rb, oa, ob = su.index_hash_float64(1), su.index_hash_float64(1), IO.RefAPI("float64"), IO.RefAPI("float64")
    for x, y in ((ra, rb), (oa, ob)):
        x.update(np.array([1.0, 2.0]), 0)
        y.update(np.array([np.nan, 1.0]), 2)
        x.merge(y)
        assert x.map_index_duplicates(np.array([1.0]), 0)[1].tolist() == [3]
        assert x.nan_count == 1
    assert not ra.has_duplicates and ra.map_index(np.array([np.nan])).tolist() == [-1]
    assert oa.has_duplicates and oa.map_index(np.array([np.nan])).tolist() == [2]
    # overflow order: merge order in the reference, row order here
    ra, rb, oa, ob = su.index_hash_int64(1), su.index_hash_int64(1), IO.RefAPI("int64"), IO.RefAPI("int64")
    for x, y in ((ra, rb), (oa, ob)):
        x.update(np.array([1, 1]), 10)
        y.update(np.array([1, 1]), 0)
        x.merge(y)
    assert ra.map_index(np.array([1])).tolist() == [10] and ra.map_index_duplicates(np.array([1]), 0)[1].tolist() == [11, 0, 1]
    assert oa.map_index(np.array([1])).tolist() == [0] and oa.map_index_duplicates(np.array([1]), 0)[1].tolist() == [1, 10, 11]


def test_deviation_masked_rows_in_duplicates():
    # the reference binds no masked map_index_duplicates (join.py's call with a mask raises TypeError); masked rows contribute none
    h = IO.RefAPI("int64")
    h.update(np.array([4, 4, 4]), 0)
    left, right = IO.IndexHash.map_index_duplicates(h, np.array([4, 4]), 0, np.array([1, 0], np.uint8))
    assert left.tolist() == [1, 1] and right.tolist() == [1, 2]


def test_index_type_from_dtype():
    # vaex/hash.py:56-60 over vaex/utils.py:754-790 with support_non_native=False
    from vaex_b200 import hash as H
    assert H.index_type_from_dtype("int32").__name__ == "index_hash_int32"
    assert H.index_type_from_dtype("datetime64[ns]").__name__ == "index_hash_int64"
    assert H.index_type_from_dtype(np.dtype(">f8")).__name__ == "index_hash_float64"
    assert H.index_type_from_dtype("uint8", transient=False, prime_growth=True).__name__ == "index_hash_uint8"
    with pytest.raises(ValueError):
        H.index_type_from_dtype(np.dtype(">i8"))
    with pytest.raises(TypeError):
        H.index_type_from_dtype("U4")
