"""The device-expression compiler (vaex_b200/expression.py) at value edges, without a GPU: its programs, run by the plain-Python
interpreter of tests/expr_oracle.py, must give numpy's answer bit for bit and numpy's dtype for every expression of the edge corpus,
and compilation must raise wherever numpy raises.  Also pins the interpreter's cast rules and numpy's correct rounding (the premise
of bit identity) to this host's numpy."""
import platform
from fractions import Fraction

import numpy as np
import pytest

import expr_oracle as EO
from helpers import same_bits
from vaex_b200 import expression as X

COLS = EO.edge_columns()
DTYPES = {k: v.dtype for k, v in COLS.items()}


def _check(expression, cols=COLS):
    """numpy raises -> compilation raises; else the program's result equals numpy's (bits, NaN payloads free; dtype)"""
    dtypes = {k: v.dtype for k, v in cols.items()}
    try:
        want = EO.numpy_eval(expression, cols)
    except Exception:
        with pytest.raises(Exception):
            X.Program(expression, dtypes)
        return "raises"
    try:
        program = X.Program(expression, dtypes)
    except NotImplementedError as e:
        assert any(w in str(e) for w in EO.UNSUPPORTED), (expression, str(e))
        return "unsupported"
    got = EO.run(program, cols)
    assert got.dtype == want.dtype, (expression, got.dtype, want.dtype)
    keep = EO.numpy_comparable(expression, cols, len(got))
    bad = np.flatnonzero(~np.array([same_bits(g, w) for g, w in zip(got[keep], want[keep])]))
    assert not len(bad), (expression, [(c[keep][bad[:4]] if len(c) else None) for c in [cols[n] for n in program.inputs]], got[keep][bad[:4]],
                          want[keep][bad[:4]])
    return "ok"


def _corpus(kind):
    exprs = EO.corpus_expressions()
    n_unary, n_binary, n_astype = 4 * 11, 10 * 121, 121
    n_lit = len(exprs) - n_unary - n_binary - n_astype - 300
    bounds = {"unary": (0, n_unary), "binary": (n_unary, n_unary + n_binary), "astype": (n_unary + n_binary, n_unary + n_binary + n_astype),
              "literals": (n_unary + n_binary + n_astype, len(exprs) - 300), "random": (len(exprs) - 300, len(exprs))}
    a, b = bounds[kind]
    assert n_lit > 0
    return exprs[a:b]


@pytest.mark.parametrize("kind", ["unary", "binary", "astype", "literals", "random"])
def test_corpus_matches_numpy(kind):
    outcomes = [_check(e) for e in _corpus(kind)]
    assert outcomes.count("ok") > len(outcomes) // 2, kind


def test_int_literal_comparisons_keep_the_literal_value():
    """a Python int outside the column's dtype is compared by its value (numpy 2), never wrapped into the dtype"""
    cols = {"u": np.array([0, 5, 255], np.uint8), "i": np.array([-2 ** 31, 0, 1, 2 ** 31 - 1], np.int32),
            "j": np.array([-2 ** 63, -1, 0, 2 ** 63 - 1], np.int64), "q": np.array([0, 2 ** 63, 2 ** 64 - 1], np.uint64)}
    for e in ["u > -1", "u == 261", "-1 < u", "i > 1099511627776", "i == 2147483648", "i != -2147483649", "j == 9223372036854775808",
              "j < 9223372036854775808", "q > -1", "q >= -9223372036854775808", "-1 == q", "q <= 18446744073709551615"]:
        assert _check(e, cols) == "ok", e


def test_literals_beyond_64_bits_compile_to_numpys_constant():
    cols = {"i": np.array([-2 ** 31, 0, 2 ** 31 - 1], np.int32), "q": np.array([0, 2 ** 63, 2 ** 64 - 1], np.uint64),
            "u": np.array([0, 3, 255], np.uint8), "j": np.array([-2 ** 63, 0, 2 ** 63 - 1], np.int64)}
    for c in cols:
        for lit in (2 ** 64, -(2 ** 63) - 1, 10 ** 30, -(10 ** 30)):
            for op in ("<", "<=", ">", ">=", "==", "!="):
                assert _check("%s %s %d" % (c, op, lit), cols) == "ok"
                assert _check("%d %s %s" % (lit, op, c), cols) == "ok"
    assert _check("(i < 18446744073709551616) & (u > 3)", cols) == "ok"


def test_signed_against_uint64_compares_exactly():
    """numpy compares a signed integer with a uint64 by value (its qQ / Qq loops), not through float64"""
    cols = {"j": np.array([2 ** 63 - 1, 2 ** 53 + 1, -1, -2 ** 63, 0, 2 ** 53], np.int64), "q": np.array([2 ** 63, 2 ** 53, 2 ** 64 - 1, 2 ** 63, 0, 2 ** 53 + 1], np.uint64),
            "i": np.array([-1, 7, 2 ** 31 - 1, -2 ** 31, 0, 5], np.int32)}
    for a, b in (("j", "q"), ("q", "j"), ("i", "q"), ("q", "i")):
        for op in ("<", "<=", ">", ">=", "==", "!="):
            assert _check("%s %s %s" % (a, op, b), cols) == "ok"
    p = X.Program("j == q", {k: v.dtype for k, v in cols.items()})
    assert p.ops[-1][1] == X.EXC_I64_U64 and all(op[0] != X.EX_CAST for op in p.ops)


def test_int_literal_to_float_rounds_like_numpy():
    """numpy converts a Python int to a double, then to float32: two roundings (2^60 + 2^36 + 1 -> 2^60)"""
    cols = {"x": np.array([2.0 ** 60, 2.0 ** 60 + 2.0 ** 37, 1.0], np.float32)}
    for e in ["x == 1152921573326323713", "x + 1152921573326323713", "x < 1152921573326323713", "x * 16777217"]:
        assert _check(e, cols) == "ok", e


def test_literal_astype_raises_like_python():
    with pytest.raises(AttributeError):
        X.Program("(3).astype('int8') + x", {"x": np.dtype("f8")})


# ---- the interpreter's cast rules against this host's numpy -------------------------------------------------------------------
INT_TARGETS = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]


@pytest.mark.skipif(platform.machine() not in ("x86_64", "AMD64"), reason="the cast rules restate numpy's x86-64 loops")
@pytest.mark.parametrize("src", ["float64", "float32"])
@pytest.mark.parametrize("target", INT_TARGETS)
def test_float_to_int_casts_match_this_hosts_numpy(src, target):
    """every float edge value to every integer type, at lengths 1, 17 and 1000 and at an odd offset.  Excluded: uint32 from NaN
    and from values outside (-2^31, 2^32), where numpy's scalar and vector loops disagree with each other (DESIGN §3)"""
    pool = EO.edge_pool(src)
    cls = X.EXC_F64 if src == "float64" else X.EXC_F32
    want_all = np.array([EO.cast(v, cls, target) for v in pool], dtype=object)

    def comparable(x):
        x = np.asarray(x, np.float64)
        return (x > -2.0 ** 31) & (x < 2.0 ** 32) if target == "uint32" else np.ones(len(x), bool)

    with np.errstate(all="ignore"):
        for k, v in enumerate(pool):  # length 1
            if comparable([v])[0]:
                assert int(np.array([v]).astype(target)[0]) == want_all[k], (v, target)
        for n in (17, 1000):
            idx = np.arange(n) % len(pool)
            for arr in (pool[idx], np.concatenate([pool[:1], pool[idx]])[1:]):  # the second starts at an odd element offset
                got = arr.astype(target)
                ok = comparable(arr)
                assert [int(g) for g in got[ok]] == list(want_all[idx][ok]), (n, target)


# ---- the premise: numpy's + - * / sqrt are correctly rounded on the float corpus ----------------------------------------------
def _round(q, dtype):
    """the exact rational q rounded to nearest-even in dtype (inf beyond the largest finite value)"""
    fi = np.finfo(dtype)
    p, emin, emax = fi.nmant + 1, fi.minexp, fi.maxexp - 1
    if q == 0:
        return Fraction(0)
    s, a = (-1 if q < 0 else 1), abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (max(e, emin) - p + 1)
    m = a / ulp
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2):
        n += 1
    r = n * ulp
    if r >= Fraction(2) ** (emax + 1):
        return None  # overflows to inf
    return s * r


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_numpy_float_arithmetic_is_correctly_rounded(dtype):
    pool = EO.edge_pool(dtype)
    pool = np.unique(pool[np.isfinite(pool)])
    a, b = np.repeat(pool, len(pool)), np.tile(pool, len(pool))
    with np.errstate(all="ignore"):
        results = {"+": a + b, "-": a - b, "*": a * b, "/": a / b}
        roots = np.sqrt(pool)
    for op, got in results.items():
        for x, y, g in zip(a.tolist(), b.tolist(), got.tolist()):
            if op == "/" and y == 0:
                continue
            fx, fy = Fraction(x), Fraction(y)
            q = fx + fy if op == "+" else fx - fy if op == "-" else fx * fy if op == "*" else fx / fy
            r = _round(q, dtype)
            if r is None:
                assert np.isinf(g) and (g > 0) == (q > 0), (x, op, y, g)
            else:
                assert Fraction(g) == r, (x, op, y, g)
    for x, g in zip(pool.tolist(), roots.tolist()):
        if x < 0:
            assert np.isnan(g) or (x == 0 and g == 0)
            continue
        # g is the nearest: the exact root lies between the midpoints to g's neighbours
        lo, hi = np.nextafter(np.array(g, dtype), -np.inf), np.nextafter(np.array(g, dtype), np.inf)
        fg = Fraction(g)
        assert ((Fraction(float(lo)) + fg) / 2) ** 2 <= Fraction(x) <= ((fg + Fraction(float(hi))) / 2) ** 2 or x == 0, (x, g)
