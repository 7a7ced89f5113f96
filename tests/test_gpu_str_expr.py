"""String calls in device expressions on the GPU (csrc/strexpr.cu through vaex_b200/expression.py): every function over numpy object,
arrow string, arrow large_string and sliced columns, with and without nulls, against the reference's golden vectors and the
restatement (tests/str_expr_oracle.py); both scan forms on both sides of their threshold; and the frame paths that evaluate them."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import str_expr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(HERE, "golden", "str_expr_golden.npz"))


def expression(name, pattern, start, end, col="s"):
    p = repr(pattern.decode("utf8"))
    if name in ("len", "byte_length"):
        return f"str_{name}({col})"
    if name == "equals2":
        return f"str_equals({col}, t)"
    if name in ("find", "rfind"):
        return f"str_{name}({col}, {p}, {start}, {end})"
    if name == "contains":
        return f"str_contains({col}, {p}, regex=False)"
    return f"str_{name}({col}, {p})"


def arrow(rows, nulls, large, sliced):
    """an arrow array over these rows' bytes (null rows keep their slots); sliced: the same rows as a slice of a longer array"""
    pre, post = ([b"head", b"", b"\xc3\xa9t"], [b"tail"]) if sliced else ([], [])
    allrows = pre + list(rows) + post
    allnulls = [False] * len(pre) + list(nulls) + [False] * len(post)
    off, data, _ = O.buffers(allrows, slack=b"")
    off = off if large else off.astype(np.int32)
    valid = pa.py_buffer(np.packbits(~np.asarray(allnulls, bool), bitorder="little")) if any(allnulls) else None
    arr = pa.Array.from_buffers(pa.large_string() if large else pa.string(), len(allrows), [valid, pa.py_buffer(off), pa.py_buffer(data)],
                                null_count=int(sum(allnulls)))
    return arr.slice(len(pre), len(rows)) if sliced else arr


def evaluate(expr, cols):
    from vaex_b200.expression import DeviceExpression
    return DeviceExpression(expr, cols).evaluate()


KINDS = ["numpy", "string", "large_string", "sliced"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("with_nulls", [False, True])
def test_every_call_against_golden_and_restatement(kind, with_nulls):
    rows, nulls = list(O.ROWS), list(O.NULLS) if with_nulls else [False] * len(O.ROWS)
    rows2, nulls2 = O.second_column()
    nulls2 = nulls2 if with_nulls else [False] * len(rows2)
    if kind == "numpy":  # a Python str holds valid UTF-8 only; a null is None with an empty slot
        keep = [i for i, r in enumerate(rows) if _utf8(r) and _utf8(rows2[i])]
        rows = [b"" if nulls[i] else rows[i] for i in keep]
        rows2 = [b"" if nulls2[i] else rows2[i] for i in keep]
        nulls, nulls2 = [nulls[i] for i in keep], [nulls2[i] for i in keep]
        cols = {"s": np.array([None if n else r.decode() for r, n in zip(rows, nulls)], dtype=object),
                "t": np.array([None if n else r.decode() for r, n in zip(rows2, nulls2)], dtype=object)}
    else:
        cols = {"s": arrow(rows, nulls, kind != "string", kind == "sliced"), "t": arrow(rows2, nulls2, kind == "large_string", False)}
    checked = 0
    for name, pattern, start, end in O.calls():
        if not _utf8(pattern):
            continue  # a pattern is a Python string literal
        want = O.evaluate(name, rows, nulls, pattern, start, O.INT64_MAX if end is None else end, rows2, nulls2)
        got = evaluate(expression(name, pattern, start, end), cols)
        assert got.dtype == want.dtype and np.array_equal(got, want), (kind, name, pattern, start, end, got, want)
        if kind != "numpy" and with_nulls:  # the very rows of the golden vectors
            assert np.array_equal(got, GOLDEN[O.key(name, pattern, start, end)]), (kind, name, pattern, start, end)
        checked += 1
    assert checked > 400


def _utf8(b):
    try:
        b.decode("utf8")
        return True
    except UnicodeDecodeError:
        return False


def test_lead_bytes_from_0xf8_step_one_byte():
    cols = {"s": arrow(O.ROWS_F8, [False] * len(O.ROWS_F8), True, False)}
    assert evaluate("str_len(s)", cols).tolist() == O.evaluate("len", O.ROWS_F8).tolist()
    for s, e in O.WINDOWS:
        want = O.evaluate("find", O.ROWS_F8, pattern=b"b", start=s, end=O.INT64_MAX if e is None else e)
        assert evaluate(f"str_find(s, 'b', {s}, {e})", cols).tolist() == want.tolist()


def _random_rows(rng, n, mean, alphabet=b"abcxyz\xc3\xa9 "):
    lens = rng.integers(0, 2 * mean + 1, n)
    pool = np.frombuffer(alphabet, np.uint8)
    data = pool[rng.integers(0, len(pool), int(lens.sum()))].tobytes()
    off = np.concatenate([[0], np.cumsum(lens)])
    return [data[off[i]:off[i + 1]] for i in range(n)]


@pytest.mark.parametrize("scan", [None, "thread", "warp"])
@pytest.mark.parametrize("mean", [4, 48, 300, 4200])
def test_scanning_calls_at_every_row_length(scan, mean, monkeypatch):
    """contains / count / find / rfind on short and long rows (>= 4 KB), in the form the call picks and in both forced forms"""
    if scan:
        monkeypatch.setenv("B200_STR_SCAN", scan)
    rng = np.random.default_rng(mean)
    n = 3000 if mean < 1000 else 300
    rows = _random_rows(rng, n, mean)
    nulls = rng.random(n) < 0.1
    cols = {"s": arrow(rows, nulls, mean % 2 == 0, True)}
    for pattern in (b"a", b"ab", b"xyz", "é".encode(), b"abcabc", b""):
        p = pattern.decode()
        cases = [("contains", f"str_contains(s, {p!r}, regex=False)", 0, None), ("find", f"str_find(s, {p!r})", 0, None),
                 ("rfind", f"str_rfind(s, {p!r})", 0, None), ("find", f"str_find(s, {p!r}, 3, -2)", 3, -2),
                 ("rfind", f"str_rfind(s, {p!r}, 2, 1000)", 2, 1000)]
        if pattern:
            cases.append(("count", f"str_count(s, {p!r})", 0, None))
        for name, e, start, end in cases:
            want = O.evaluate(name, rows, nulls, pattern, start, O.INT64_MAX if end is None else end)
            got = evaluate(e, cols)
            assert np.array_equal(got, want), (scan, mean, e)


def _words(n, seed=0):
    rng = np.random.default_rng(seed)
    words = np.array(["Amsterdam", "Hamburg", "Augsburg", "Berlin", "", "Århus", "NL", "Alkmaar", None], dtype=object)
    return words[rng.integers(0, len(words), n)], rng


@pytest.mark.parametrize("kind", ["numpy", "string", "large_string"])
def test_frame_filter_selection_groupby_and_binby(kind):
    from vaex_b200 import agg
    from vaex_b200.execution import Executor
    from vaex_b200.frame import Frame
    n = 20_000
    w, rng = _words(n)
    x = rng.standard_normal(n)
    k = rng.integers(0, 5, n)
    s = w if kind == "numpy" else pa.array(w.tolist(), pa.string() if kind == "string" else pa.large_string())
    cols = dict(name=s, city=s, x=x, k=k)
    sv = np.array([v if v is not None else "" for v in w], dtype=object)
    isnull = np.array([v is None for v in w])
    starts_a = np.array([v.startswith("A") for v in sv])
    burg = np.array(["burg" in v for v in sv])
    nl = (sv == "NL") & ~isnull
    for ex in (None, Executor(nthreads=3, chunk_size=1111)):  # several workers, chunks that end mid-word groups
        df = Frame(cols, executor=ex)
        assert df.filter("str_startswith(name, 'A')").count() == starts_a.sum()
        assert df.count(selection="str_equals(city, 'NL')") == nl.sum()
        assert df.count(selection="city == 'NL'") == nl.sum()
        assert list(df.count(selection=["city == 'NL'", "city != 'NL'"])) == [nl.sum(), n - nl.sum()]
        np.testing.assert_allclose(df.filter("str_contains(city, 'burg', regex=False)").sum("x"), x[burg].sum(), rtol=1e-12)
        # a string filter and a string groupby key on one frame: the key set and the grid see the kept rows only
        out = df.filter("str_contains(city, 'burg', regex=False)").groupby("city", agg="count", sort=True)
        assert out["city"].tolist() == ["Augsburg", "Hamburg"]
        assert out["count"].tolist() == [int((sv[burg] == "Augsburg").sum()), int((sv[burg] == "Hamburg").sum())]
        out = df.filter("str_len(name) > 2").groupby("k", agg=[agg.count(), agg.sum("x")], sort=True)
        lens = np.array([len(v) for v in sv])
        keep = lens > 2
        assert out["k"].tolist() == sorted(set(k[keep].tolist()))
        assert out["count"].tolist() == [int((k[keep] == v).sum()) for v in out["k"]]
        # str_len as a binby: mean of x per string length
        lens_b = np.array([len(v) for v in sv])  # the corpus' words are single code points per character
        got = df.mean("x", binby="str_len(name)", limits=[0, 64], shape=64)
        for L in range(12):
            sel = lens_b == L
            if sel.any():
                np.testing.assert_allclose(got[L], x[sel].mean(), rtol=1e-12)
        assert np.array_equal(df.evaluate("str_byte_length(name)"), np.array([len(v.encode()) for v in sv]))


def test_ten_million_rows_against_the_restatement():
    rng = np.random.default_rng(7)
    n = 10_000_000
    lens = rng.integers(0, 17, n)
    pool = np.frombuffer(b"abcdefgh", np.uint8)
    data = pool[rng.integers(0, len(pool), int(lens.sum()))]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    arr = pa.Array.from_buffers(pa.large_string(), n, [None, pa.py_buffer(off), pa.py_buffer(data)])
    raw = data.tobytes()
    rows = [raw[off[i]:off[i + 1]] for i in range(n)]
    cols = {"s": arr}
    assert np.array_equal(evaluate("str_byte_length(s)", cols), lens)
    assert np.array_equal(evaluate("str_startswith(s, 'ab')", cols), np.array([r.startswith(b"ab") for r in rows]))
    assert np.array_equal(evaluate("str_count(s, 'a')", cols), np.array([r.count(b"a") for r in rows]))
    assert np.array_equal(evaluate("str_rfind(s, 'ba', 1)", cols), O.evaluate("rfind", rows, pattern=b"ba", start=1))


def test_binby_expressions_are_device_columns():
    """a binby expression that is not a column, numeric or string, bins like the same values given as a column; the aggregation
    methods and the legacy statistic methods take it alike"""
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(3)
    n = 50_000
    x, y, z = rng.standard_normal(n), rng.standard_normal(n), rng.standard_normal(n)
    w, _ = _words(n, 1)
    lens = np.array([0 if v is None else len(v) for v in w], np.int64)
    df = Frame(dict(x=x, y=y, z=z, s=pa.array(w.tolist())))
    ref = Frame(dict(x=x, y=y, z=z, x2=x * 2, n=lens))
    for expr, col, lim in (("x * 2", "x2", [-4, 4]), ("str_len(s)", "n", [0, 16])):
        assert np.array_equal(df.count(binby=expr, limits=lim, shape=16), ref.count(binby=col, limits=lim, shape=16))
        # float sums: the same rows in every cell, added in an order the device's atomics choose
        np.testing.assert_allclose(df.sum("y", binby=[expr, "z"], limits=[lim, [-2, 2]], shape=8),
                                   ref.sum("y", binby=[col, "z"], limits=[lim, [-2, 2]], shape=8), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(df.cov("y", "z", binby=expr, limits=lim, shape=8), ref.cov("y", "z", binby=col, limits=lim, shape=8),
                                   rtol=1e-9, atol=1e-12)
