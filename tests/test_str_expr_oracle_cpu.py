"""The string-call restatement (tests/str_expr_oracle.py) against the compiled, unmodified reference (oracle/_ref/strfunc_shim) over
the edge corpus, and the golden vectors the GPU tests read against both."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import str_expr_oracle as O  # noqa: E402

REF = os.path.join(HERE, "..", "oracle", "_ref")


@pytest.fixture(scope="module")
def shim():
    sys.path.insert(0, REF)
    try:
        import strfunc_shim
    except ImportError:
        pytest.skip("oracle/_ref/strfunc_shim is built only where the reference sources are")
    return strfunc_shim


@pytest.mark.parametrize("sliced", [False, True])
def test_restatement_matches_the_reference(shim, sliced):
    """every call of the corpus; sliced: the reference reads offsets that do not start at 0 (an arrow slice's)"""
    import make_golden_str_expr as G
    rows, nulls = O.ROWS, O.NULLS
    for name, pattern, start, end in O.calls():
        if sliced:
            off, data, mask = O.buffers([b"skip me"] + rows, [False] + nulls)
            off, mask = off[1:], mask[1:]
            if name == "equals2":
                continue  # equals2 takes the rotated column, checked unsliced
            want = {"notequals": lambda: ~np.asarray(shim.equals(off, data, mask, pattern)),
                    "len": lambda: np.asarray(shim.len(off, data, mask)), "byte_length": lambda: np.asarray(shim.byte_length(off, data, mask)),
                    "find": lambda: np.asarray(shim.find(off, data, mask, pattern, start, end, True)),
                    "rfind": lambda: np.asarray(shim.find(off, data, mask, pattern, start, end, False))}.get(name)
            if name in ("contains", "count"):
                continue
            got_ref = want() if want else np.asarray(getattr(shim, name)(off, data, mask, pattern))
        else:
            got_ref = G.reference(shim, name, pattern, start, end)
        rows2, nulls2 = O.second_column()
        mine = O.evaluate(name, rows, nulls, pattern, start, O.INT64_MAX if end is None else end, rows2, nulls2)
        assert got_ref.dtype == mine.dtype, (name, pattern)
        assert np.array_equal(got_ref, mine), (name, pattern, start, end, got_ref, mine)


def test_contains_and_count_match_bytes_find_and_count():
    for p in O.PATTERNS:
        assert O.evaluate("contains", O.ROWS, pattern=p).tolist() == [r.find(p) >= 0 for r in O.ROWS]
        if p:
            assert O.evaluate("count", O.ROWS, pattern=p).tolist() == [r.count(p) for r in O.ROWS]


def test_multibyte_sequence_cut_off_at_the_end_counts_once(shim):
    rows = [b"ab\xe2\x82", b"\xf0\x9f\x98", b"\xc3", "€".encode()[:1], b"a\xf0"]
    off, data, _ = O.buffers(rows)
    assert np.asarray(shim.len(off, data, None)).tolist() == [3, 1, 1, 1, 2] == O.evaluate("len", rows).tolist()


def test_lead_bytes_from_0xf8_step_one_byte():
    """the reference never ends on them (DESIGN.md §1): the restatement, like the device, steps one byte"""
    assert O.evaluate("len", O.ROWS_F8).tolist() == [1, 3, 2, 2]
    assert O.find(b"\xf8ab", b"b", 1) == 1 and O.find(b"\xf8ab", b"b", 0, -1) == -1 and O.find(b"\xf8ab", b"a", 0, -1) == 1


def test_golden_vectors_are_the_reference_s():
    g = np.load(os.path.join(HERE, "golden", "str_expr_golden.npz"))
    rows2, nulls2 = O.second_column()
    for name, pattern, start, end in O.calls():
        want = O.evaluate(name, O.ROWS, O.NULLS, pattern, start, O.INT64_MAX if end is None else end, rows2, nulls2)
        got = g[O.key(name, pattern, start, end)]
        assert got.dtype == want.dtype and np.array_equal(got, want), (name, pattern, start, end)
