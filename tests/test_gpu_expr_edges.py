"""Device expressions, filters and filter compaction (csrc/expr.cu, vaex_b200/expression.py) at value edges: the edge corpus of
tests/expr_oracle.py on the device against the plain-Python interpreter and numpy, filtered frames and selections whose masks
depend on the literal / mixed-sign / cast rules, `expression.compact` at its block and scan boundaries, `_ordinal_values` at edge
keys, and the program limits."""
import numpy as np
import pytest

import expr_oracle as EO
from helpers import same_bits, to_device

pytestmark = pytest.mark.gpu

COLS = EO.edge_columns()
DTYPES = {k: v.dtype for k, v in COLS.items()}


def _dev(a):
    """a device copy of a numpy column that keeps its dtype (unsigned types included)"""
    from vaex_b200.expression import DeviceArray
    t = to_device(a)
    return DeviceArray(t.data_ptr(), len(a), a.dtype, keep=t)


def _cases():
    """(expression, program, oracle result) for every corpus expression the compiler accepts (the CPU suite checks the rest)"""
    from vaex_b200 import expression as X
    if not hasattr(_cases, "memo"):
        out = []
        for e in EO.corpus_expressions():
            try:
                p = X.Program(e, DTYPES)
            except Exception:
                continue
            out.append((e, p, EO.run(p, COLS)))
        _cases.memo = out
    return _cases.memo


def _evaluate(expression, cols):
    from vaex_b200.expression import DeviceExpression
    return DeviceExpression(expression, cols).evaluate()


@pytest.mark.parametrize("memory", ["host", "device", "mixed"])
def test_corpus_on_the_device(memory):
    names = list(COLS)
    cols = {k: (_dev(v) if memory == "device" or (memory == "mixed" and n % 2) else v) for n, (k, v) in enumerate(COLS.items())}
    for e, p, want in _cases():
        got = _evaluate(e, cols)
        assert got.dtype == want.dtype, e
        assert same_bits(got, want), (e, np.flatnonzero(~np.array([same_bits(g, w) for g, w in zip(got, want)]))[:5])
    assert len(names) == 11


def test_corpus_over_more_than_one_grid_sweep():
    """1,100,003 rows: more than one sweep of k_eval's grid-stride loop (132 SMs x 16 blocks x 256 threads), device columns that
    start at an odd element offset; against the interpreter (tiled) and numpy"""
    n = 1_100_003
    big = {k: np.resize(v, n) for k, v in COLS.items()}
    cols = {k: _dev(np.concatenate([v[:1], v]))[1:] for k, v in big.items()}
    cases = _cases()
    for e, p, want in cases[::9] + [c for c in cases if c[0] in ("i8 == u8", "u8 < i8", "f8.astype('int8')", "f4.astype('uint64')")]:
        got = _evaluate(e, cols)
        assert same_bits(got, np.resize(want, n)), e
        ref = EO.numpy_eval(e, big)
        keep = EO.numpy_comparable(e, big, n)
        assert got.dtype == ref.dtype and same_bits(got[keep], ref[keep]), e


# the expressions whose masks the literal / mixed-sign / cast rules decide
FILTERS = ["u > -1", "u == 261", "(u == 5) | (i > 1099511627776)", "i == 2147483648", "j == 9223372036854775808", "i < 18446744073709551616",
           "-9223372036854775809 >= j", "j == q", "j < q", "x.astype('int8') == 0", "x.astype('uint64') > 9223372036854775808",
           "x.astype('int32') == -2147483648", "x.astype('uint16') != 0"]


def _frame_columns(n, seed=7):
    rng = np.random.default_rng(seed)
    cols = {"u": rng.integers(0, 256, n).astype("u1"), "i": rng.integers(-2 ** 31, 2 ** 31, n).astype("i4"),
            "j": rng.integers(-2 ** 62, 2 ** 62, n), "q": rng.integers(0, 2 ** 64 - 1, n, dtype=np.uint64),
            "x": rng.normal(0, 1e3, n), "y": rng.integers(-3, 3, n) + 0.5}
    # edge rows only in chunks 3 and 7 (6000-row chunks): the other chunks keep no row under most filters
    for lo in (18_000, 42_000):
        s = slice(lo, lo + 6000, 3)
        k = len(range(lo, lo + 6000, 3))
        cols["j"][s] = np.resize(np.array([2 ** 63 - 1, 2 ** 53 + 1, -2 ** 63, -1], np.int64), k)
        cols["q"][s] = np.resize(np.array([2 ** 63, 2 ** 53, 2 ** 63, 2 ** 64 - 1], np.uint64), k)
        cols["u"][s] = 5
        cols["i"][s] = np.resize(np.array([-2 ** 31, 2 ** 31 - 1], np.int32), k)
        cols["x"][s] = np.resize(np.array([3e9 + 1, 1.5e19, 2.0 ** 64, np.nan, np.inf, -np.inf, 2.0 ** 63 + 6144, -0.0, 65536.5, 2.0 ** 31]), k)
    return cols


@pytest.mark.parametrize("device", [False, True])
def test_filters_and_selections_at_edges(device, oracle):
    from vaex_b200 import execution
    from vaex_b200.frame import Frame
    n = 60_000
    cols = _frame_columns(n)
    src = dict(cols, x=to_device(cols["x"]), y=to_device(cols["y"])) if device else cols
    df = Frame(src, executor=execution.Executor(nthreads=2, chunk_size=6_000))
    lim = [[-3, 3]]
    for f in FILTERS:
        keep = EO.evaluate(f, cols)
        assert np.array_equal(keep, EO.numpy_eval(f, cols)), f
        y = cols["y"][keep]
        want_count = oracle.binby([oracle.scalar(y, -3, 3, 16)], [oracle.agg("count")])[0]
        fdf = df.filter(f)
        assert np.array_equal(fdf.count(binby=["y"], limits=lim, shape=16, edges=True), want_count), f
        want_sum = oracle.binby([oracle.scalar(y, -3, 3, 16)], [oracle.agg("sum", y)])[0]
        assert np.array_equal(fdf.sum("y", binby=["y"], limits=lim, shape=16, edges=True), want_sum), f  # halves: exact sums
        sel = df.count(binby=["y"], limits=lim, shape=16, selection=f, edges=True)
        assert np.array_equal(sel, oracle.binby([oracle.scalar(cols["y"], -3, 3, 16)], [oracle.agg("count", cols["y"], mask=keep.astype("u1"))])[0]), f
        if keep.any():
            assert np.array_equal(fdf.minmax("y", raw=True), oracle.minmax(y, raw=True)), f
            out = fdf.groupby("u").agg({"y": "count"})
            order = np.argsort(np.asarray(out["u"]))
            ks, cs = np.unique(cols["u"][keep], return_counts=True)
            assert np.array_equal(np.asarray(out["u"])[order], ks), f
            assert np.array_equal(np.asarray(out["count"])[order], cs), f
    # at least one filter keeps every row, one none, one only rows of the two edge chunks
    kept = [int(EO.evaluate(f, cols).sum()) for f in FILTERS]
    assert n in kept and 0 in kept and any(0 < k < 12_000 for k in kept)


# ---- expression.compact -------------------------------------------------------------------------------------------------------
LENGTHS = [1, 1023, 1024, 1025, 2 ** 20, 2 ** 20 + 1, 3 * 2 ** 20 + 7]
PATTERNS = ["none", "all", "first", "last", "alternate", "random"]


def _keep(pattern, n, rng):
    """uint8 keep bytes; non-zero (2..255 here, never just 1) means keep"""
    k = np.zeros(n, np.uint8)
    if pattern == "all":
        k[:] = rng.integers(2, 256, n)
    elif pattern == "first":
        k[0] = 200
    elif pattern == "last":
        k[-1] = 2
    elif pattern == "alternate":
        k[1::2] = 255
    elif pattern == "random":
        k[:] = rng.integers(0, 256, n) * (rng.random(n) < 0.5)
    return k


@pytest.mark.parametrize("n", LENGTHS)
def test_compact_lengths_patterns_and_memory(n):
    from vaex_b200 import expression
    rng = np.random.default_rng(n)
    dts = ["u1", "i2", "i4", "f8"] * 4  # 16 columns, itemsize 1, 2, 4 and 8
    cols = [rng.integers(-2 ** 31, 2 ** 31, n).astype(dt) if np.dtype(dt).kind != "f" else rng.standard_normal(n) for dt in dts]
    for k, pattern in enumerate(PATTERNS):
        keep = _keep(pattern, n, rng)
        memory = ["host", "device", "mixed"][k % 3]
        if memory == "host":
            inp, km = cols, keep
        else:  # device inputs sliced at an odd element offset
            dev = [_dev(np.concatenate([c[:1], c]))[1:] for c in cols]
            inp = dev if memory == "device" else [d if j % 2 else c for j, (c, d) in enumerate(zip(cols, dev))]
            km = _dev(np.concatenate([keep[:1], keep]))[1:] if memory == "device" else keep
        count, out = expression.compact(0, km, inp)
        want = keep != 0
        assert count == int(want.sum()), (n, pattern, memory)
        for c, o in zip(cols, out):
            assert same_bits(o.to_numpy(), c[want]), (n, pattern, memory, c.dtype)


def test_compact_refuses_seventeen_columns():
    from vaex_b200 import expression
    cols = [np.arange(10, dtype="i4")] * 17
    with pytest.raises(Exception, match="b200_compact"):
        expression.compact(0, np.ones(10, np.uint8), cols)


# ---- _ordinal_values at edge keys -----------------------------------------------------------------------------------------------
KEY_DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8"]


@pytest.mark.parametrize("dtype", KEY_DTYPES)
def test_ordinal_values_at_edge_keys(dtype):
    """sets holding the dtype's edge values (INT64_MIN; -1, whose sign-extended pattern is the table's empty sentinel; 2^64-1; NaN
    payloads; -0.0 and +0.0 as distinct members), probed with those keys and with keys that are not members (-> -1)"""
    from oracle import oracle as O
    from vaex_b200 import hash as vhash
    from vaex_b200.frame import Frame
    pool = EO.edge_pool(dtype)
    _, first = np.unique(pool.view("u%d" % pool.dtype.itemsize), return_index=True)
    distinct = pool[np.sort(first)]  # distinct bit patterns, in pool order
    if dtype.startswith("float"):  # one NaN member: the set keeps a single NaN slot
        nan = np.isnan(distinct)
        distinct = np.concatenate([distinct[~nan][:-3], distinct[nan][:1], distinct[~nan][-3:]])
    members = distinct[:-3]  # the last three are not members
    hm = vhash.HashMapUnique(np.dtype(dtype))
    hm.add(members)
    ref = O.OrderedSet(dtype)
    ref.update(members)
    probe = np.resize(pool, 1001)
    got = Frame({"k": probe}, variables={"hm": hm}).evaluate("_ordinal_values(k, hm)")
    want = ref.map_ordinal(probe)
    assert got.dtype == want.dtype and np.array_equal(got, want), dtype
    assert (want == -1).any()
    if dtype.startswith("float"):  # an integer column probing a float set: the compiler casts the keys first
        ints = np.resize(np.array([0, 1, -1, 3_000_000, 2 ** 31 - 1, -2 ** 31, 16777217], np.int64), 1001)
        got = Frame({"k": ints}, variables={"hm": hm}).evaluate("_ordinal_values(k, hm)")
        assert np.array_equal(got, ref.map_ordinal(ints.astype(dtype))), dtype


@pytest.mark.parametrize("size", [127, 128, 32767, 32768])
def test_ordinal_dtype_follows_the_set_size(size):
    from oracle import oracle as O
    from vaex_b200 import hash as vhash
    from vaex_b200.frame import Frame
    for dtype in ("int64", "float32"):
        members = np.concatenate([EO.edge_pool(dtype)[:5], np.arange(size - 5) + 10]).astype(dtype)
        assert len(np.unique(members.view("u%d" % members.dtype.itemsize))) == size
        hm = vhash.HashMapUnique(np.dtype(dtype))
        hm.add(members)
        ref = O.OrderedSet(dtype)
        ref.update(members)
        probe = np.concatenate([members[::-1], np.array([-5, 7, 9], dtype)])
        got = Frame({"k": probe}, variables={"hm": hm}).evaluate("_ordinal_values(k, hm)")
        want = ref.map_ordinal(probe)
        assert got.dtype == want.dtype == np.dtype("int8" if size < 128 else "int16" if size < 32768 else "int32"), (dtype, size)
        assert np.array_equal(got, want), (dtype, size)


# ---- program limits -------------------------------------------------------------------------------------------------------------
def test_program_limits():
    """stack depth 12 and 64 ops evaluate; depth 13 and 65 ops raise, never return a value"""
    from vaex_b200 import expression as X
    cols = {"a": COLS["f8"], "b": COLS["i4"]}

    def nested(k):  # right-nested sums: stack depth k
        return "a" if k == 1 else "a + (%s)" % nested(k - 1)

    def chain(nops):  # -a + a + a + ...: stack depth 2, one negation when the op count is even
        operands = (nops + 1) // 2
        return "-" * (nops - (2 * operands - 1)) + " + ".join(["a"] * operands)

    for e, depth, nops in [(nested(12), 12, 23), (chain(64), 2, 64)]:
        p = X.Program(e, {k: v.dtype for k, v in cols.items()})
        assert EO.stack_depth(p.ops) == depth and len(p.ops) == nops, e
        got = _evaluate(e, cols)
        assert same_bits(got, EO.run(p, cols)) and same_bits(got, EO.numpy_eval(e, cols)), e
    for e, depth, nops in [(nested(13), 13, 25), (chain(65), 2, 65)]:
        p = X.Program(e, {k: v.dtype for k, v in cols.items()})
        assert EO.stack_depth(p.ops) == depth and len(p.ops) == nops, e
        with pytest.raises(Exception, match="b200_eval"):
            _evaluate(e, cols)
