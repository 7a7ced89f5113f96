"""Frame.sort and Frame.take on the device: the reference's sort tests (sort_cases.py), the edge corpus of sort_oracle.py through
b200_argsort against pa.compute.sort_indices element for element, the radix passes each key layout runs, filters, expression keys,
take's arguments and placement, a 1e8-row sort against torch.sort, and the row limit and memory refusals."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import sort_cases  # noqa: E402
import sort_oracle as S  # noqa: E402

pytestmark = pytest.mark.gpu


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


def values(frame, name):
    """a column's values over the frame's filtered rows"""
    col = frame.columns[name]
    v = host_values(frame.evaluate(name) if getattr(col, "device_virtual", False) else col)
    if frame._filter_expression is not None:
        keep = frame.evaluate(frame._filter_expression)
        v = [x for x, k in zip(v, keep) if k]
    return v


def make_frame(columns, filter=None, place="host"):
    import torch
    from vaex_b200.frame import Frame
    if place == "device":
        columns = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and not np.ma.isMaskedArray(v) and v.dtype.kind in "biuf"
                   and v.dtype.isnative else v for k, v in columns.items()}
    return Frame(columns, pin=place == "pinned", filter=filter)


# ---- the reference's cases ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("place", ["host", "device", "pinned"])
@pytest.mark.parametrize("case", sorted(sort_cases.CASES))
def test_reference_cases(case, place):
    columns, filter, kwargs, want = sort_cases.CASES[case]
    df = make_frame(columns, filter, place)
    out = df.sort(**kwargs)
    for name, expected in want.items():
        assert values(out, name) == expected, (name, values(out, name))
    if case == "empty":
        assert out._filter_expression == filter  # a frame without passing rows comes back as a copy, filter kept
    else:
        assert out._filter_expression is None and len(out) == len(want["x"])


def test_ascending_list_length():
    df = make_frame({"x": np.arange(3), "y": np.arange(3)})
    with pytest.raises(AssertionError, match='If "ascending" is a list, it must have the same number of elements as "by".'):
        df.sort(["x", "y"], ascending=[True])
    # a flag ascends only when it `is True`, as the reference's `order is True`
    assert values(df.sort("x", ascending=1), "x") == [2, 1, 0]


# ---- the corpus through b200_argsort --------------------------------------------------------------------------------------------
def corpus_frame(keys, place):
    """keys of sort_oracle -> a frame with columns k0.. and `row`, on the host or (plain native numeric keys) on the device"""
    import torch
    from vaex_b200.frame import Frame
    columns = {}
    for i, (v, m, _) in enumerate(keys):
        if v.dtype.kind == "O":
            v = np.array([None if (m is not None and mm) else x for x, mm in zip(v, m if m is not None else [False] * len(v))], dtype=object)
            columns[f"k{i}"] = v
        elif m is not None:
            columns[f"k{i}"] = np.ma.array(v, mask=m)
        elif place == "device" and v.dtype.kind in "biuf" and v.dtype.isnative:
            columns[f"k{i}"] = torch.from_numpy(v).cuda()
        else:
            columns[f"k{i}"] = v
    columns["row"] = np.arange(len(keys[0][0]))
    return Frame(columns)


def check_corpus(keys, place="host"):
    df = corpus_frame(keys, place)
    out = df.sort([f"k{i}" for i in range(len(keys))], ascending=[not d for _, _, d in keys])
    got, want = np.asarray(values(out, "row")), S.arrow_argsort(keys)
    assert np.array_equal(got, want), (got.tolist(), want.tolist())


@pytest.mark.parametrize("place", ["host", "device"])
@pytest.mark.parametrize("dtype", S.NUMERIC + S.TIMES + ["string"])
def test_corpus_one_key(dtype, place):
    rng = np.random.default_rng(len(dtype))
    for masked in (False, True):
        for byteswap in (False, True):
            for descending in (False, True):
                check_corpus([S.random_key(rng, dtype, 500, masked, byteswap, descending)], place)


@pytest.mark.parametrize("place", ["host", "device"])
def test_corpus_many_keys(place):
    rng = np.random.default_rng(3)
    kinds = S.NUMERIC + S.TIMES + ["string"]
    for trial in range(60):
        n = int(rng.integers(1, 400))
        keys = [S.random_key(rng, rng.choice(kinds), n, rng.random() < 0.4, rng.random() < 0.3, rng.random() < 0.5) for _ in range(rng.integers(1, 5))]
        check_corpus(keys, place)


def test_stable_when_all_equal():
    for descending in (False, True):
        check_corpus([(np.zeros(3000, "f4"), None, descending), (np.ones(3000, "i8"), None, not descending)])


# ---- which passes each key layout runs ------------------------------------------------------------------------------------------------
# name -> (keys as (values, mask, descending), words (k_sort_encode launches), radix passes (k_radix_scatter launches))
def path_cases():
    rng = np.random.default_rng(11)
    n = 100_000
    small = rng.integers(0, 256, n).astype("i4")
    return {
        # one byte varies; no class field (no NaN or null possible)
        "int32 small": ([(small, None, False)], 1, 1),
        # a mask adds the class field above the value, and a null row's value bits are zero where the others have the flipped
        # sign bit: bytes 0, 3 and 4 vary
        "int32 masked": ([(small, rng.random(n) < 0.1, False)], 1, 3),
        # two int32 keys packed into one word: byte 0 of the last key, byte 4 of the first
        "two int32 packed": ([(small, None, False), (small[::-1].copy(), None, True)], 1, 2),
        # float64 0..255: value bytes 5-7 vary (word 1); word 2 holds its class bit and the int32 (bits 1-8: bytes 0 and 1)
        "int32 then float64": ([(small, None, False), (small.astype("f8"), None, False)], 2, 5),
        # float32 {1, 2}: value bytes 2 and 3; no NaN, so the class byte is skipped
        "float32 without NaN": ([(rng.choice(np.array([1.0, 2.0], "f4"), n), None, False)], 1, 2),
        # with NaN the class byte is sorted too
        "float32 with NaN": ([(rng.choice(np.array([1.0, 2.0, np.nan], "f4"), n), None, False)], 1, 3),
        # nothing varies: no pass at all
        "all equal": ([(np.full(n, 7, "i8"), None, False)], 1, 0),
    }


def _record_paths(path):
    """run every path case under torch.profiler and write the kernel counts (a fresh process: late in a long pytest process the
    profiler's sessions come back without kernel records more and more often)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, (keys, _, _) in path_cases().items():
        df = corpus_frame(keys, "host")
        cols = [f"k{i}" for i in range(len(keys))]
        asc = [not d for _, _, d in keys]
        df.sort(cols, ascending=asc)  # warm-up: module load, string sets
        for attempt in range(2):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                res = df.sort(cols, ascending=asc)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
            if names:
                break
        row = np.asarray(values(res, "row"))
        out[name] = {"encode": sum("k_sort_encode" in x for x in names), "scatter": sum("k_radix_scatter" in x for x in names),
                     "correct": bool(np.array_equal(row, S.arrow_argsort(keys))), "kernels": len(names)}
    with open(path, "w") as f:
        json.dump(out, f)


@pytest.fixture(scope="module")
def paths(tmp_path_factory):
    out = tmp_path_factory.mktemp("prof") / "sort_paths.json"
    subprocess.check_call([sys.executable, os.path.abspath(__file__), str(out)], cwd=os.path.dirname(HERE))
    return json.loads(out.read_text())


@pytest.mark.parametrize("name", sorted(path_cases()))
def test_radix_passes(paths, name):
    _, words, passes = path_cases()[name]
    got = paths[name]
    assert got["kernels"] > 0, "torch.profiler recorded no CUDA kernel"
    assert got["correct"], name
    assert (got["encode"], got["scatter"]) == (words, passes), got


# ---- filters and expression keys --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("place", ["host", "device"])
def test_filtered(place):
    rng = np.random.default_rng(5)
    n = 5000
    x = rng.standard_normal(n)
    x[::97] = np.nan
    y = rng.integers(0, 20, n)
    df = make_frame({"x": x, "y": y, "row": np.arange(n)}, "y < 12", place)
    out = df.sort(["y", "x"], ascending=[False, True])
    keep = y < 12
    want = np.flatnonzero(keep)[S.arrow_argsort([(y[keep], None, True), (x[keep], None, False)])]
    assert values(out, "row") == want.tolist()
    assert out._filter_expression is None
    # filtered down to no row: a copy with the filter
    empty = make_frame({"x": x, "y": y}, "y > 100", place).sort("x")
    assert empty._filter_expression == "y > 100" and values(empty, "x") == []


@pytest.mark.parametrize("place", ["host", "device"])
def test_virtual_and_expression_keys(place):
    rng = np.random.default_rng(6)
    n = 3000
    a, b = rng.integers(-50, 50, n).astype("i4"), rng.standard_normal(n).astype("f4")
    df = make_frame({"a": a, "b": b, "row": np.arange(n)}, None, place)
    df.add_virtual_column("v", "a * 2 - b")
    out = df.sort(["v"], ascending=False)
    v = a * np.float32(2) - b
    assert values(out, "row") == S.arrow_argsort([(v, None, True)]).tolist()
    assert getattr(out.columns["v"], "device_virtual", False)  # stays virtual over the gathered columns
    assert np.allclose(values(out, "v"), v[np.asarray(values(out, "row"))])
    out = df.sort(["-a", "b"])
    assert values(out, "row") == S.arrow_argsort([(-a, None, False), (b, None, False)]).tolist()


# ---- take ---------------------------------------------------------------------------------------------------------------------------
def take_frame(place):
    import pyarrow as pa
    rng = np.random.default_rng(8)
    n = 200
    cols = {"a": rng.standard_normal(n), "b": np.ma.array(rng.integers(0, 9, n).astype("i4"), mask=rng.random(n) < 0.2),
            "s": pa.array([None if i % 7 == 0 else f"s{i}" for i in range(n)]), "t": np.arange(n).astype("M8[s]"), "d": rng.integers(0, 1000, n)}
    df = make_frame(cols, "a > -0.5", place)
    df.add_virtual_column("v", "d + 1")
    return df, cols


@pytest.mark.parametrize("place", ["host", "device"])
@pytest.mark.parametrize("filtered", [True, False])
@pytest.mark.parametrize("dropfilter", [True, False])
def test_take(place, filtered, dropfilter):
    df, cols = take_frame(place)
    keep = cols["a"] > -0.5
    rows = np.flatnonzero(keep)
    idx = np.array([3, 0, 0, 17, 5, len(rows) - 1])
    out = df.take(idx, filtered=filtered, dropfilter=dropfilter)
    src = rows[idx] if filtered else idx
    sel = keep[src] if not dropfilter else np.ones(len(src), bool)
    for name in ("a", "b", "t", "d"):
        want = np.ma.asarray(cols[name])[src][sel].tolist() if name != "t" else cols["t"][src][sel].tolist()
        assert values(out, name) == want, name
    assert values(out, "s") == [cols["s"][int(i)].as_py() for i in src[sel]]
    assert values(out, "v") == (cols["d"][src][sel] + 1).tolist()
    assert (out._filter_expression is None) == dropfilter
    # placement: device columns stay, host ones come back, strings as arrow, masks kept
    from vaex_b200 import _lib
    assert _lib.is_device(out.columns["d"]) == (place == "device")
    assert np.ma.isMaskedArray(out.columns["b"]) and type(out.columns["s"]).__module__.startswith("pyarrow")


@pytest.mark.parametrize("kind", ["i1", "i2", "i4", "i8", "u1", "u2", "u4", "u8", "list", "torch-i8", "torch-i4", "torch-u1"])
def test_take_index_kinds(kind):
    import torch
    df = make_frame({"x": np.arange(100) * 10})
    idx = [5, 99, 0, 42]
    if kind == "list":
        index = idx
    elif kind.startswith("torch"):
        index = torch.tensor(idx, dtype={"i8": torch.int64, "i4": torch.int32, "u1": torch.uint8}[kind[-2:]], device="cuda")
    else:
        index = np.array(idx, kind)
    assert values(df.take(index), "x") == [i * 10 for i in idx]


def test_take_empty_and_out_of_range():
    import torch
    df = make_frame({"x": np.arange(10), "s": np.array(["a"] * 10, dtype=object)}, "x > 4")
    assert values(df.take([]), "x") == [] and values(df.take([]), "s") == []
    for bad in ([-1], [5], np.array([2 ** 63], "u8"), torch.tensor([7], device="cuda")):
        with pytest.raises(IndexError, match="out of bounds for 5 rows"):
            df.take(bad)
    with pytest.raises(IndexError, match="out of bounds for 10 rows"):
        df.take([10], filtered=False)
    assert values(df.take([9], filtered=False, dropfilter=True), "x") == [9]


# ---- scale, limits -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float32", "int64"])
def test_1e8_device_rows_against_torch(dtype):
    """1e8 device rows: for these dtypes (no NaN, no -0.0 drawn) the encoded order is the values' order, so torch's stable sort
    gives the same permutation"""
    import torch
    from vaex_b200 import _lib
    from vaex_b200 import sort as _sort
    n = 10 ** 8
    g = torch.Generator(device="cuda").manual_seed(1)
    if dtype == "float32":
        x = torch.randn(n, device="cuda", generator=g)
        x[x == 0] = 1.0
    else:
        x = torch.randint(-2 ** 40, 2 ** 40, (n,), device="cuda", generator=g, dtype=torch.int64)
    want = torch.sort(x, stable=True).indices
    perm = _sort.argsort([_sort.Key(x, _lib.DTYPE_CODE[dtype])], n)
    assert torch.equal(perm, want)
    perm = _sort.argsort([_sort.Key(x, _lib.DTYPE_CODE[dtype], descending=True)], n)
    assert torch.equal(perm, torch.sort(x, stable=True, descending=True).indices)


def test_row_limit_before_allocation():
    from vaex_b200 import _lib
    from vaex_b200 import sort as _sort

    class Huge:
        __cuda_array_interface__ = {"shape": (2 ** 32,), "typestr": "<i4", "data": (0, False), "version": 3, "strides": None}

        def __len__(self):
            return 2 ** 32
    before = _lib.context().mem_stats()["live"]
    with pytest.raises(ValueError, match="exceed the limit of 4294967295 rows"):
        _sort.argsort([_sort.Key(Huge(), _lib.I32)], 2 ** 32)
    assert _lib.context().mem_stats()["live"] == before


def test_memory_error(monkeypatch):
    from vaex_b200 import _lib
    from vaex_b200 import sort as _sort
    df = make_frame({"x": np.arange(1000)[::-1].copy()})
    before = _lib.context().mem_stats()["live"]
    monkeypatch.setattr(_sort, "free_bytes", lambda device: 1000)
    with pytest.raises(MemoryError, match=r"\(%d bytes\) exceed the 1000 bytes free" % _sort.scratch_bytes(1000)):
        df.sort("x")
    assert _lib.context().mem_stats()["live"] == before


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _record_paths(sys.argv[1])
