"""Compiling the string calls of device expressions (vaex_b200/expression.py): result dtypes, the programs and every refusal."""
import numpy as np
import pyarrow as pa
import pytest

from vaex_b200 import expression as X

DT = {"s": np.dtype("O"), "t": np.dtype("O"), "x": np.dtype("f8"), "i": np.dtype("i4"), "a": np.dtype("O")}
STRINGS = ["s", "t"]


def compile_(e):
    return X.Program(e, DT, strings=STRINGS)


@pytest.mark.parametrize("expression,dtype,call", [
    ("str_equals(s, 'NL')", "bool", (X.EX_STR_EQUALS, ("s",), b"NL")),
    ("s == 'NL'", "bool", (X.EX_STR_EQUALS, ("s",), b"NL")),
    ("'NL' == s", "bool", (X.EX_STR_EQUALS, ("s",), b"NL")),
    ("str_equals('NL', s)", "bool", (X.EX_STR_EQUALS, ("s",), b"NL")),
    ("str_equals(s, t)", "bool", (X.EX_STR_EQUALS2, ("s", "t"), b"")),
    ("s == t", "bool", (X.EX_STR_EQUALS2, ("s", "t"), b"")),
    ("str_startswith(s, 'A')", "bool", (X.EX_STR_STARTSWITH, ("s",), b"A")),
    ("str_endswith(s, pat='é')", "bool", (X.EX_STR_ENDSWITH, ("s",), "é".encode())),
    ("str_contains(s, 'burg', regex=False)", "bool", (X.EX_STR_CONTAINS, ("s",), b"burg")),
    ("str_contains(s, 'burg')", "bool", (X.EX_STR_CONTAINS, ("s",), b"burg")),
    ("str_count(s, 'ab')", "int64", (X.EX_STR_COUNT, ("s",), b"ab")),
    ("str_count(s, 'ab', regex=True)", "int64", (X.EX_STR_COUNT, ("s",), b"ab")),
    ("str_find(s, 'a')", "int64", (X.EX_STR_FIND, ("s",), b"a")),
    ("str_rfind(s, 'a')", "int64", (X.EX_STR_RFIND, ("s",), b"a")),
    ("str_len(s)", "int64", (X.EX_STR_LEN, ("s",), b"")),
    ("str_byte_length(s)", "int64", (X.EX_STR_BYTE_LENGTH, ("s",), b"")),
])
def test_result_dtype_and_call(expression, dtype, call):
    p = compile_(expression)
    assert p.dtype == np.dtype(dtype)
    assert [c.key()[:3] for c in p.strcalls] == [call]
    assert p.ops == [(X.EX_INPUT, X._cls(dtype), 0, 0.0, 0)]  # the call's column is the program's one input


def test_notequals_is_not_equals():
    for e in ("str_notequals(s, 'x')", "str_notequals('x', s)", "s != 'x'", "'x' != s", "s != t"):
        p = compile_(e)
        assert p.dtype == np.bool_ and p.ops[-1][0] == X.EX_NOT, e


def test_find_window_arguments():
    assert compile_("str_find(s, 'a', 2, -1)").strcalls[0].key() == (X.EX_STR_FIND, ("s",), b"a", 2, -1)
    assert compile_("str_rfind(s, sub='a', start=-3, end=None)").strcalls[0].key() == (X.EX_STR_RFIND, ("s",), b"a", -3, (1 << 63) - 1)


def test_string_call_inputs_follow_the_column_inputs():
    p = compile_("(str_len(s) > i) & (x < 1) & str_startswith(t, 'a') & (str_len(s) < 9)")
    assert p.inputs == ["i", "x"]
    assert [c.key()[:2] for c in p.strcalls] == [(X.EX_STR_LEN, ("s",)), (X.EX_STR_STARTSWITH, ("t",))]  # the repeated call runs once
    reads = sorted({arg for op, _, arg, _, _ in p.ops if op == X.EX_INPUT})
    assert reads == [0, 1, 2, 3]


def test_numeric_programs_are_unchanged():
    assert X.Program("x * 2 + i", DT).ops == compile_("x * 2 + i").ops
    assert compile_("x * 2 + i").strcalls == []


@pytest.mark.parametrize("bad", ["s + 1", "s < 'a'", "-s", "str_len(x)", "str_len(a)", "str_len(i + 1)", "'a'", "s == 1", "s == x",
                                 "str_startswith(s, t)", "str_find(s, 'a', x)", "str_contains(s, 'a', regex=x)", "str_equals(x, 'a')",
                                 "str_equals('a', x)", "str_equals('a', 'b')", "str_lower(s)", "sqrt(s)"])
def test_refusals(bad):
    with pytest.raises(NotImplementedError):
        compile_(bad)


@pytest.mark.parametrize("pattern", [".", "^a", "a$", "a*", "a+", "a?", "(a)", "[a]", "{1}", "a|b", "\\\\d"])
def test_regex_patterns_are_refused(pattern):
    with pytest.raises(NotImplementedError, match="regex"):
        compile_(f"str_contains(s, '{pattern}')")
    with pytest.raises(NotImplementedError, match="regex"):
        compile_(f"str_count(s, '{pattern}', regex=True)")
    assert compile_(f"str_contains(s, '{pattern}', regex=False)").dtype == np.bool_


def test_empty_count_pattern_is_refused():
    """in both of the reference's branches: the literal one never ends, the regex one is not computed here"""
    for e in ("str_count(s, '')", "str_count(s, '', regex=False)", "str_count(s, '', regex=True)"):
        with pytest.raises(ValueError, match="empty pattern"):
            compile_(e)


def test_wrong_arguments():
    with pytest.raises(TypeError):
        compile_("str_len(s, 'a')")
    with pytest.raises(TypeError):
        compile_("str_startswith(s)")


def test_device_expression_tells_strings_from_arrow_numerics():
    """arrow strings and numpy object / unicode strings are string columns; an arrow numeric column is not"""
    for col in (pa.array(["a", None]), pa.array(["a", "b"], pa.large_string()), np.array(["a", None], dtype=object), np.array(["a", "b"])):
        assert X.DeviceExpression("str_len(s)", {"s": col}).dtype == np.int64
    with pytest.raises(NotImplementedError, match="not supported in device expressions"):
        X.DeviceExpression("str_len(s)", {"s": pa.array([1, 2])})
    with pytest.raises(NotImplementedError, match="not supported in device expressions"):
        X.DeviceExpression("s + 1", {"s": pa.array(["a", "b"])})
    e = X.DeviceExpression("str_len(s) + x", {"s": pa.array(["a", "b"]), "x": np.zeros(2)})
    assert len(e) == 2 and len(e.columns) == 2


def test_too_many_inputs():
    dt = {f"s{k}": np.dtype("O") for k in range(9)}
    with pytest.raises(NotImplementedError, match="more than 8"):
        X.Program(" + ".join(f"str_len(s{k})" for k in range(9)), dt, strings=list(dt))


def test_a_chunk_stages_only_its_own_bytes():
    """a slice of a long arrow column shares the column's buffer: what goes to the device is the slice's byte range, indexed by its
    own offsets shifted back by offsets[0] (string calls and filter compaction of string columns)"""
    from vaex_b200.join import _string_source
    col = pa.array([f"row{i:06d}" + "x" * (i % 7) for i in range(10_000)], pa.large_string())
    for arr in (col, col.cast(pa.string())):
        part = arr.slice(5_000, 10)
        offsets, isz, data, first, mask = _string_source(part)
        assert isz == (8 if arr.type == pa.large_string() else 4) and mask is None
        assert len(data) == offsets[-1] - offsets[0] == sum(len(v.as_py()) for v in part)
        assert [bytes(data[offsets[i] - first:offsets[i + 1] - first]).decode() for i in range(10)] == part.to_pylist()
    with_nulls = pa.array(["a", None, "bcd", None, "e"] * 100).slice(101, 7)
    offsets, _, data, first, mask = _string_source(with_nulls)
    assert mask.tolist() == [1, 0, 1, 0, 0, 1, 0] and len(data) == offsets[-1] - offsets[0]
