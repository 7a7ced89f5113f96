"""Frame.join and the b200_take / b200_take_strings gathers on the device, against the join restatement (join_oracle.py)."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import join_cases  # noqa: E402
import join_oracle as J  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = ["float64", "float32", "int64", "int32", "int16", "int8", "uint64", "uint32", "uint16", "uint8", "bool", "datetime64[ns]"]


def host_values(col):
    """a frame column as a python list, None = missing"""
    import pyarrow as pa
    if isinstance(col, (pa.Array, pa.ChunkedArray)):
        return col.to_pylist()
    if hasattr(col, "__cuda_array_interface__") and not isinstance(col, np.ndarray):
        import torch
        from vaex_b200 import _lib
        _lib.context().sync()
        col = torch.as_tensor(col, device="cuda").cpu().numpy()
    if np.ma.isMaskedArray(col):
        return col.tolist()
    return np.asarray(col).tolist()


def values(frame, name, filtered=True):
    col = frame.columns[name]
    if getattr(col, "device_virtual", False):
        col = frame.evaluate(name)
    v = host_values(col)
    if filtered and frame._filter_expression is not None:
        keep = frame.evaluate(frame._filter_expression)
        v = [x for x, k in zip(v, keep) if k]
    return v


def same(a, b):
    def eq(x, y):
        if isinstance(x, float) and isinstance(y, float) and math.isnan(x) and math.isnan(y):
            return True
        return x == y
    return len(a) == len(b) and all(eq(x, y) for x, y in zip(a, b))


def to_frame(spec, place="host", nthreads=None, chunk_size=None):
    """a case frame on the host, page-locked or with its plain numeric columns on the device"""
    import torch
    from vaex_b200 import execution
    from vaex_b200.frame import Frame
    columns, filter = spec
    if place == "device":
        columns = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and not np.ma.isMaskedArray(v) and v.dtype.kind in "biuf"
                   else v for k, v in columns.items()}
    ex = execution.Executor(nthreads, chunk_size=chunk_size)
    return Frame(columns, executor=ex, filter=filter, pin=place == "pinned")


def check_against_oracle(got, want, filtered=True):
    assert set(got.columns) == set(want.columns)
    for name in want.columns:
        assert same(values(got, name, filtered), want.values(name, filtered)), name


@pytest.mark.parametrize("place", ["host", "device"])
@pytest.mark.parametrize("case", join_cases.CASES, ids=[c[0] for c in join_cases.CASES])
def test_reference_case(case, place):
    _, left, right, kwargs, expected = case
    got = to_frame(left, place).join(to_frame(right, place), **kwargs)
    for name, want in expected.items():
        if name == "__names__":
            assert set(got.columns) == want
        else:
            assert same(values(got, name), want), (name, values(got, name), want)
    oracle = J.join(J.OFrame(left[0], join_cases.filter_mask(*left)), J.OFrame(right[0], join_cases.filter_mask(*right)), **kwargs)
    check_against_oracle(got, oracle, filtered=False)


@pytest.mark.parametrize("case", join_cases.ERRORS, ids=[c[0] for c in join_cases.ERRORS])
def test_reference_error(case):
    _, left, right, kwargs, exc, text = case
    with pytest.raises(exc, match=text):
        to_frame(left).join(to_frame(right), **kwargs)


def test_string_key_error():
    left = to_frame(({"s": np.array(["a", "b"], dtype=object), "x": np.arange(2)}, None))
    right = to_frame(({"s": np.array(["a", "c"], dtype=object), "y": np.arange(2)}, None))
    with pytest.raises(TypeError, match="index_hash_string"):
        left.join(right, on="s")


def random_keys(rng, dtype, n, distinct):
    dt = np.dtype(dtype)
    if dt.kind == "b":
        return rng.integers(0, 2, n).astype(bool)
    if dt.kind == "M":
        return (np.datetime64("2020-01-01", "ns") + rng.integers(0, distinct, n) * np.timedelta64(3600, "s")).astype(dt)
    if dt.kind == "f":
        k = rng.integers(0, distinct, n).astype(dt)
        k[rng.random(n) < 0.05] = np.nan
        return k
    hi = min(distinct, np.iinfo(dt).max)
    return rng.integers(0, hi, n).astype(dt)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("how", ["left", "inner", "right"])
@pytest.mark.parametrize("dup", [False, True])
def test_random_join(dtype, how, dup):
    rng = np.random.default_rng(abs(hash((dtype, how, dup))) % 2**32)
    n_left, n_right = 3000, 500 if dup else 60
    distinct = 80
    lk = random_keys(rng, dtype, n_left, distinct)
    if dup:
        rk = random_keys(rng, dtype, n_right, distinct)
    else:
        rk = np.unique(random_keys(rng, dtype, 4 * n_right, distinct))[:n_right]
        rk = rk[~np.isnan(rk)] if rk.dtype.kind == "f" else rk
        rng.shuffle(rk)
    lmask = rng.random(n_left) < 0.1
    rmask = rng.random(len(rk)) < 0.1 if not dup else rng.random(len(rk)) < 0.05
    if not dup:
        rmask[:] = False
    left = {"k": np.ma.array(lk, mask=lmask), "v": rng.standard_normal(n_left), "lx": rng.integers(0, 1000, n_left).astype("i4")}
    right = {"k": np.ma.array(rk, mask=rmask), "w": np.ma.array(rng.standard_normal(len(rk)), mask=rng.random(len(rk)) < 0.2),
             "s": np.array([None if i % 7 == 3 else "s%d" % i for i in range(len(rk))], dtype=object), "rx": np.arange(len(rk)).astype("u2")}
    lfilter = "lx < 700"
    for nthreads, chunk in ((1, None), (8, 256)):
        for rfilter in (None, "rx > 5"):
            if how == "right" and rfilter is not None:
                continue
            kwargs = dict(on="k", how=how, rsuffix="_r", allow_duplication=True)
            got = to_frame((left, lfilter), nthreads=nthreads, chunk_size=chunk).join(to_frame((right, rfilter), nthreads=nthreads, chunk_size=chunk), **kwargs)
            want = J.join(J.OFrame(left, join_cases.filter_mask(left, lfilter)), J.OFrame(right, join_cases.filter_mask(right, rfilter)), **kwargs)
            check_against_oracle(got, want, filtered=False)


@pytest.mark.parametrize("place", ["host", "pinned", "device"])
def test_placement(place):
    """a device left key gives device columns when every key matches; a missing row gives a host np.ma column"""
    rng = np.random.default_rng(5)
    rk = rng.permutation(1000).astype("i8")
    lk = rng.integers(0, 1000, 20000).astype("i8")
    right = {"k": rk, "w": rng.standard_normal(1000), "c": rng.integers(0, 9, 1000).astype("i2")}
    left = {"k": lk, "v": np.arange(20000)}
    frames = [to_frame((left, None), place), to_frame((right, None), place)]
    try:
        check_placement(place, frames, right, lk, rk)
    finally:
        for f in frames:  # page-locked columns are unregistered before numpy frees them
            if f._pinned is not None:
                f._pinned.release()


def check_placement(place, frames, right, lk, rk):
    import torch
    got = frames[0].join(frames[1], on="k")
    if place == "device":
        assert isinstance(got.columns["w"], torch.Tensor) and got.columns["w"].is_cuda
    else:
        assert isinstance(got.columns["w"], np.ndarray) and not np.ma.isMaskedArray(got.columns["w"])
    inv = np.empty(1000, np.int64)
    inv[rk] = np.arange(1000)
    assert np.array_equal(np.asarray(values(got, "w")), right["w"][inv[lk]])
    # aggregations on the joined frame
    assert np.array_equal(got.count(binby="c", limits=[-0.5, 8.5], shape=9), np.bincount(right["c"][inv[lk]], minlength=9))
    g = got.groupby("c", agg="count", sort=True)
    assert np.array_equal(np.asarray(g["c"]), np.arange(9)) and np.array_equal(np.asarray(g["count"]), np.bincount(right["c"][inv[lk]], minlength=9))
    # a key without a match: that column becomes a host masked array
    lk2 = lk.copy()
    lk2[::10] = 5000
    frames.append(to_frame(({"k": lk2}, None), place))
    got = frames[-1].join(frames[1], on="k")
    assert np.ma.isMaskedArray(got.columns["w"]) and got.columns["w"].mask.sum() == 2000


def test_virtual_columns_and_variables():
    """test_join_virtual_columns / test_join_variables: the right's virtual columns are gathered with their values, expression keys work"""
    left = to_frame(({"j": np.array([444, 5]), "x": np.array([1, 2]), "y": np.array([2, 3])}, None))
    left.add_virtual_column("z", "x + y")
    right = to_frame(({"j": np.array([5, 444]), "x": np.array([2, 4]), "yy": np.array([3, 1])}, None))
    right.add_virtual_column("z", "x + yy")
    right.variables["yes"] = 3
    out = left.join(right, on="j", rprefix="r_", rsuffix="_rhs")
    assert values(out, "z") == [3, 5]
    assert values(out, "r_z_rhs") == [5, 5]
    assert values(out, "r_x_rhs") == [4, 2]
    assert out.variables["yes"] == 3
    out = left.join(right, left_on="x * 2", right_on="x", rsuffix="_r")
    assert values(out, "yy") == [3, 1]
    joined = left.join(right, on="j", rsuffix="_r")
    again = left.join(joined, on="j", rsuffix="_rr")  # a joined frame as the right side (test_join_indexed)
    assert values(again, "yy") == [1, 3]


def take_call(index, columns, src_len, device=False):
    from vaex_b200 import join
    return join.take(index, columns, src_len, device)


@pytest.mark.parametrize("isz", [1, 2, 4, 8])
@pytest.mark.parametrize("device", [False, True])
def test_take_widths(isz, device):
    import torch
    rng = np.random.default_rng(isz)
    n_src = 100
    idx = rng.integers(-1, n_src, 5000).astype(f"i{isz}")
    cols = [(rng.integers(0, 255, n_src).astype(f"u{k}"), None) for k in (1, 2, 4, 8)]
    cols.append((rng.standard_normal(n_src), rng.random(n_src) < 0.3))
    index = torch.from_numpy(idx).cuda() if device else idx
    out = take_call(index, cols, n_src, device)
    for (src, mask), (vals, valid) in zip(cols, out):
        vals = np.asarray(host_values(vals))
        missing = (idx < 0) | (mask[np.maximum(idx, 0)] if mask is not None else False)
        assert valid is not None
        assert np.array_equal(np.asarray(host_values(valid)) == 0, missing)
        assert np.array_equal(vals[idx >= 0], src[idx[idx >= 0]])
        assert np.all(vals[idx < 0] == 0)


def test_take_edges():
    from vaex_b200 import join
    src = np.arange(10.)
    with pytest.raises(RuntimeError, match="source length"):
        join.take(np.array([0, 10], np.int64), [(src, None)], 10, False)
    assert len(join.take(np.zeros(0, np.int64), [(src, None)], 10, False)[0][0]) == 0
    cols = [(src * k, None) for k in range(16)]
    out = join.take(np.array([3, 1], np.int32), cols, 10, False)
    assert all(np.array_equal(o, [3. * k, 1. * k]) and v is None for k, (o, v) in enumerate(out))
    out = join.take(np.array([3, 1], np.int32), cols + cols[:3], 10, False)
    assert len(out) == 19


@pytest.mark.parametrize("large", [False, True])
def test_take_strings(large):
    import pyarrow as pa
    import torch
    from vaex_b200 import join
    data = ["", "a", None, "hello world, a longer string " * 5, "x" * 33, "", "é", None, "last"]
    arr = pa.array(data, type=pa.large_string() if large else pa.string())
    for src, ref in ((arr, data), (arr.slice(2, 5), data[2:7])):
        idx = np.array([0, -1, len(ref) - 1, 1, 2, 3, 4, 3, 0], np.int64)
        for index in (idx, torch.from_numpy(idx).cuda()):
            out, missing = join.take_strings(index, src)
            want = [ref[i] if i >= 0 else None for i in idx]
            assert out.to_pylist() == want
            assert missing == any(w is None for w in want)
    with pytest.raises(RuntimeError, match="source length"):
        join.take_strings(np.array([len(data)], np.int64), arr)
    empty, _ = join.take_strings(np.zeros(0, np.int64), arr)
    assert len(empty) == 0


def test_large_join_against_numpy():
    """1e8 left rows against 1e6 right rows with duplicates, on the device, against an argsort join"""
    import torch
    rng = np.random.default_rng(11)
    n_left, n_right = 100_000_000, 1_000_000
    rk = rng.integers(0, 900_000, n_right).astype(np.int32)
    lk = rng.integers(0, 1_000_000, n_left).astype(np.int32)
    w = rng.integers(0, 1 << 30, n_right).astype(np.int64)
    left = {"k": torch.from_numpy(lk).cuda()}
    right = {"k": torch.from_numpy(rk).cuda(), "w": torch.from_numpy(w).cuda()}
    got = to_frame((left, None), "host").join(to_frame((right, None), "host"), on="k", allow_duplication=True)
    lrows, rrows = J.numpy_join(lk, rk)
    col = got.columns["w"]
    assert np.ma.isMaskedArray(col) and len(col) == len(lrows)
    want_mask = rrows < 0
    assert np.array_equal(np.ma.getmaskarray(col), want_mask)
    assert np.array_equal(np.ma.getdata(col)[~want_mask], w[rrows[~want_mask]])
    k = host_values(got.columns["k"])
    assert np.array_equal(np.asarray(k), lk[lrows])
