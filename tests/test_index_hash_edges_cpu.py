"""The restatement of index_hash<T> (tests/index_hash_oracle.py) on the index edge corpus (tests/index_hash_edge_cases.py): against the
committed answers of the compiled reference (index_hash_edges_golden.npz) and against the compiled classes where oracle/_ref exists,
in both of its key modes; and what the golden file covers."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import index_hash_edge_cases as E  # noqa: E402
import index_hash_oracle as IO  # noqa: E402
import make_golden_index_hash as G  # noqa: E402
import make_golden_index_hash_edges as GE  # noqa: E402
import set_cases as S  # noqa: E402


def assert_same(got, want, name):
    assert set(got) == set(want), name
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), f"{name}: {k}"


@pytest.fixture(scope="module")
def golden():
    return GE.load()


@pytest.mark.parametrize("bits", [False, True])
def test_golden_against_restatement(golden, bits):
    assert len(golden) == len(GE.cases()) == 2 * len(GE.KINDS) * len(E.DTYPES)
    for name, (case, res) in golden.items():
        assert_same(G.run(lambda dt: IO.classes(dt, bits), case), res, name)


def test_golden_inputs_are_the_corpus(golden):
    cases = GE.cases()
    assert set(cases) == set(golden)
    for name, case in cases.items():
        got = golden[name][0]
        assert len(got["updates"]) == len(case["updates"]) and len(got["merges"]) == len(case["merges"]), name
        for (k1, m1, s1), (k2, m2, s2) in zip(got["updates"] + [m[0] for m in got["merges"]], case["updates"] + [m[0] for m in case["merges"]]):
            assert k1.dtype == k2.dtype and np.array_equal(k1.view(f"u{k1.itemsize}"), k2.view(f"u{k2.itemsize}")) and s1 == s2, name
            assert (m1 is None) == (m2 is None) and (m1 is None or np.array_equal(m1, m2)), name
        assert np.array_equal(got["lookup"].view(f"u{got['lookup'].itemsize}"), case["lookup"].view(f"u{case['lookup'].itemsize}")), name


def test_golden_covers_the_corpus(golden):
    assert {c["dtype"] for c, _ in golden.values()} == set(E.DTYPES)
    for kind in GE.KINDS:  # every kind of case meets every nmaps
        assert {c["nmaps"] for n, (c, _) in golden.items() if n.startswith(kind + "_")} == set(E.NMAPS), kind
    for dtype in E.DTYPES:
        dt = np.dtype(dtype)
        mine = [(c, r) for c, r in golden.values() if c["dtype"] == dtype]
        inserted = np.concatenate([k for c, _ in mine for k, _, _ in c["updates"] + [u for m in c["merges"] for u in m]])
        looked_up = np.concatenate([c["lookup"] for c, _ in mine])
        bits = lambda a: set(a.view(f"u{dt.itemsize}").tolist())  # noqa: E731
        s = S.sentinel(dt)
        if s is not None:
            assert s in inserted and s in looked_up, dtype
            # the sentinel has duplicates, so its overflow rows reach map_index_duplicates
            assert any(np.count_nonzero(k == s) > 1 for c, _ in mine for k, _, _ in c["updates"]), dtype
        edges = S.edge_values(dt, zeros=False)
        assert bits(edges) <= bits(inserted) and bits(edges) <= bits(looked_up), dtype
        nans = S.nan_values(dt)
        assert bits(nans) <= bits(inserted) and bits(nans) <= bits(looked_up), dtype
        if dt.kind == "f":
            assert not (np.signbit(inserted) & (inserted == 0)).any(), "-0.0 is left out of the golden file"
            assert any(r["scalars"][3] for _, r in mine)  # NaN rows
        assert any(r["scalars"][4] for _, r in mine)  # null rows
        assert any(c["lookup_mask"] is not None for c, _ in mine) and any(c["lookup_mask"] is None for c, _ in mine)
        assert any(c["merges"] for c, _ in mine) and any(len(c["updates"]) > 1 for c, _ in mine)
        if dt.kind != "b":  # keys never inserted, through every width
            assert all(any(r["unknown_" + w] for _, r in mine) for w in G.WIDTHS), dtype


def test_unordered_cases_cover_the_edges():
    cases = E.all_unordered()
    for dtype in E.DTYPES:
        mine = [c for c in cases.values() if c["dtype"] == dtype]
        starts = [s for c in mine for _, _, s in c["updates"] + [u for m in c["merges"] for u in m]]
        assert min(starts) < 0 and max(starts) + 100 > 2 ** 40
        spans = set()
        for c in mine:
            rows = [(s, s + len(k) - 1) for k, _, s in c["updates"]]
            spans.add(max(r[1] for r in rows) - min(r[0] for r in rows))
        assert set(E.SPANS) <= spans, dtype
        assert {c["nmaps"] for c in mine} >= set(E.NMAPS) - {32767}


def test_restatement_against_compiled_reference(ref):
    """the whole dtype x nmaps product of the sequential cases, of which the golden file stores a rotation"""
    su = ref.modules()[1]
    cases = E.all_sequential(zeros=False)
    assert len(cases) == len(GE.KINDS) * len(E.DTYPES) * len(E.NMAPS)
    for name, case in cases.items():
        want = G.run(lambda dt: getattr(su, "index_hash_" + dt), case)
        assert_same(G.run(IO.classes, case), want, name)
        assert_same(G.run(lambda dt: IO.classes(dt, True), case), want, name)


def test_bit_pattern_mode_splits_signed_zeros():
    """the default keys by value (-0.0 == 0.0, the reference's std::equal_to); bit-pattern mode, the device's rule, keeps them apart"""
    keys = np.array([0.0, 1.0, -0.0])
    h = IO.RefAPI("float64")
    h.update(keys, 0)
    assert h.map_index(np.array([-0.0, 0.0])).tolist() == [0, 0] and h.count == 2 and h.has_duplicates
    b = IO.RefAPI("float64", 1, bits=True)
    b.update(keys, 0)
    assert b.map_index(np.array([-0.0, 0.0])).tolist() == [2, 0] and b.count == 3 and not b.has_duplicates


def test_bit_pattern_mode_casts_lookups_by_value():
    h = IO.IndexHash("float64", bits=True)
    h.update(np.array([1.5, -1.0, np.inf]), None, 4)
    rows, unknown = h.map_index(np.array([1.5, -1.0, np.inf, 2.0], np.float32))
    assert rows.tolist() == [4, 5, 6, -1] and unknown
    h = IO.IndexHash("int64", bits=True)
    h.update(np.array([-1, 2 ** 63 - 1]), None, 0)
    assert h.map_index(np.array([-1, 7], np.int8))[0].tolist() == [0, -1]


def test_nan_payloads_share_one_row():
    for dtype in ("float32", "float64"):
        nans = S.nan_values(dtype)
        for bits in (False, True):
            h = IO.IndexHash(dtype, bits=bits)
            h.update(np.concatenate([np.ones(1, dtype), nans]), None, 0)
            assert h.nan_count == len(nans) and h.count == 2
            assert h.map_index(nans)[0].tolist() == [len(nans)] * len(nans)


def test_nat_is_an_ordinary_int64_key(ref):
    """a join indexes datetimes as index_hash_int64 over their int64 ticks: NaT is INT64_MIN there, an ordinary key that finds the other
    NaT rows (not a NaN or a null), next to the other int64 extremes"""
    su = ref.modules()[1]
    ticks = np.array(["NaT", "1970-01-01", "NaT", "2262-04-11T23:47:16.854775807", "1677-09-21T00:12:43.145224193"], "M8[ns]").view(np.int64)
    assert ticks[0] == np.iinfo(np.int64).min and ticks[3] == np.iinfo(np.int64).max
    look = np.array([ticks[0], ticks[3], ticks[4], -1, 0])
    for h in (su.index_hash_int64(1), IO.RefAPI("int64", 1, bits=True)):
        h.update(ticks, 10)
        assert (h.nan_count, h.null_count, h.has_duplicates, h.count) == (0, 0, True, 4)
        assert h.map_index(look).tolist() == [10, 13, 14, -1, 11]
        assert np.asarray(h.map_index_duplicates(look, 0)[1]).tolist() == [12]
