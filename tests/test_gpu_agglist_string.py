"""AggList_string_int64 on the device: golden parity with the compiled reference, the reference's own list-of-strings tests restated
on Frame, a chunked multi-worker run against the oracle, device-resident and sliced inputs, and an output past 2^32 bytes."""
import numpy as np
import pytest

import agglist_string_cases as cases
from oracle.agglist_string import agg_list_string

pytestmark = pytest.mark.gpu


def _superagg_binners(setup):
    from vaex_b200 import superagg
    bs = []
    for kind, data, arg in setup["binners"]:
        if kind == "ordinal":
            bs.append(getattr(superagg, "BinnerOrdinal_" + data.dtype.name)(1, "x", arg, 0, False, False))
        else:
            bs.append(getattr(superagg, "BinnerScalar_" + data.dtype.name)(1, "y", arg[0], arg[1], int(arg[2])))
    return bs


@pytest.mark.parametrize("setup_name", cases.SETUPS)
def test_golden_parity_through_superagg(setup_name):
    """the generator's bin() calls replayed through the mirror: list offsets, string offsets, bytes and validity bit-identical"""
    import pyarrow as pa
    from vaex_b200 import superagg
    setup = cases.load()[setup_name]
    strs = cases.strings_of(setup)
    arrow = pa.array(strs, type=pa.large_string())
    for k, (name, case) in enumerate(sorted(setup["cases"].items())):
        bs = _superagg_binners(setup)
        g = superagg.Grid(bs)
        a = superagg.AggList_string_int64(g, 1, 1, case["dropnan"], case["dropnull"])
        for i1, i2 in setup["calls"]:
            for b, (_, data, _) in zip(bs, setup["binners"]):
                b.set_data(0, np.ascontiguousarray(data[i1:i2]))
            # the input kinds string_buffers takes, in turn: sliced large_string (offsets[0] != 0), sliced string, a list
            a.set_data(0, [arrow[i1:i2], arrow[i1:i2].cast(pa.string()), strs[i1:i2]][k % 3], 0)
            if case["masked"]:
                a.set_data_mask(0, setup["valid"][i1:i2])
            else:
                a.clear_data_mask(0)
            g.bin(0, [a], i2 - i1)
        lo, so, by, va = a.result_arrays()
        assert np.array_equal(lo, case["list_offsets"]), name
        assert np.array_equal(so, case["str_offsets"]), name
        assert np.array_equal(by, case["str_bytes"]), name
        assert np.array_equal(va, case["str_valid"]), name
        got = a.get_result()
        assert str(got.type) == "large_list<item: large_string>" and len(got) == len(g)
        assert got.flatten().to_pylist() == [None if not v else bytes(by[so[i]:so[i + 1]]).decode() for i, v in enumerate(va)]


@pytest.mark.parametrize("dropmissing", [False, True])
@pytest.mark.parametrize("by_col_has_missing", [False, True])
@pytest.mark.parametrize("combine", [False, True])
def test_groupby_agg_list_string(dropmissing, by_col_has_missing, combine):
    # tests/agg_test.py:663-694 (test_agg_list) of the reference, its string column: groupby('id').agg(list(food, dropmissing=...))
    import pyarrow as pa
    from vaex_b200 import agg
    from vaex_b200.frame import Frame
    ids = np.ma.array([1, 2, 2, 1, 1, 3, 3], mask=[0, 0, 0, 0, 0, by_col_has_missing, by_col_has_missing], dtype="i8")
    food = pa.array(["cake", "apples", "oranges", "meat", "meat", "carrots", None])
    cols = dict(id=ids, food=food)
    by = "id"
    if combine:  # the sparse path: a second, constant key
        cols["one"] = np.zeros(7, "i4")
        by = ["id", "one"]
    out = Frame(cols).groupby(by, agg=[agg.list("food", dropmissing=dropmissing)], combine=combine, sort=True)
    if dropmissing:
        assert out["food_list"].to_pylist() == [["cake", "meat", "meat"], ["apples", "oranges"], ["carrots"]]
    else:
        assert out["food_list"].to_pylist() == [["cake", "meat", "meat"], ["apples", "oranges"], ["carrots", None]]
    assert out["id"].tolist() == ([1, 2, None] if by_col_has_missing else [1, 2, 3])


def test_agg_arrow_list_of_strings():
    # tests/agg_test.py:711-714 (test_agg_arrow): list(df.s) per integer group; plus string keys and Frame.list
    import pyarrow as pa
    from vaex_b200 import agg
    from vaex_b200.frame import Frame
    s = ["aap", "aap", "noot", "mies", None, "mies", "kees", "mies", "aap"]
    x = np.array([0, 0, 0, 0, 0, 1, 1, 1, 2], "i8")
    df = Frame(dict(x=x, s=pa.array(s)))
    out = df.groupby("x", agg={"s": agg.list("s")}, sort=True)
    assert out["x"].tolist() == [0, 1, 2]
    assert set(out["s"].to_pylist()[0]) == {"mies", "aap", "noot", None}
    assert out["s"].to_pylist() == [["aap", "aap", "noot", "mies", None], ["mies", "kees", "mies"], ["aap"]]
    # string keys: every group lists its own key, the null group a null
    out = df.groupby("s", agg={"l": agg.list("s")}, sort=True)
    assert out["s"].tolist() == ["aap", "kees", "mies", "noot", None]
    assert out["l"].to_pylist() == [["aap"] * 3, ["kees"], ["mies"] * 3, ["noot"], [None]]
    df.categorize("x", 0, 3)
    lists = df.list("s", binby="x", dropmissing=True)
    assert lists.to_pylist() == [["aap", "aap", "noot", "mies"], ["mies", "kees", "mies"], ["aap"], [], []]


@pytest.mark.parametrize("nthreads", [1, 3])
def test_frame_list_string_chunked_against_the_oracle(nthreads):
    """~1e6 rows, ~1e4 groups, chunks fed by 1 or 3 workers: exactly the oracle's lists with one worker (arrival = row order),
    the same multiset per cell with three (chunks arrive in completion order)"""
    import pyarrow as pa
    from oracle import oracle as O
    from vaex_b200.execution import Executor
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(31)
    n, groups = 1_000_003, 10_000
    k = rng.integers(0, groups, n).astype("i4")
    vocab = np.array(["", "é", "x" * 40] + [f"w{i}-" + "z" * (i % 23) for i in range(997)], dtype=object)
    strs = vocab[rng.integers(0, len(vocab), n)]
    strs[rng.random(n) < 0.05] = None
    df = Frame(dict(k=k, s=pa.array(strs.tolist(), type=pa.string())), executor=Executor(nthreads=nthreads, chunk_size=65_537))
    df.categorize("k", 0, groups)
    got = df.list("s", binby="k")
    want_lo, want_so, want_by, want_va = agg_list_string(k, strs.tolist(), groups + 2)
    lo = np.asarray(got.offsets)
    assert np.array_equal(lo, want_lo)
    flat = got.flatten()
    if nthreads == 1:
        _, so, by = flat.buffers()
        so = np.frombuffer(so, np.int64, count=len(flat) + 1, offset=flat.offset * 8)
        assert np.array_equal(so - so[0], want_so)
        assert np.array_equal(np.frombuffer(by, np.uint8)[so[0]:so[-1]], want_by)
        assert np.array_equal(np.asarray(flat.is_valid()), want_va.astype(bool))
    else:
        mine = flat.to_pylist()
        want = [None if not v else bytes(want_by[want_so[i]:want_so[i + 1]]).decode() for i, v in enumerate(want_va)]
        key = lambda s: (s is None, s or "")  # noqa: E731
        for c in range(groups + 2):
            assert sorted(mine[lo[c]:lo[c + 1]], key=key) == sorted(want[lo[c]:lo[c + 1]], key=key), c


def _device_strings(strs):
    import torch
    from oracle import ref_driver as R
    off, by, nulls = R.pack_strings(strs)
    return torch.from_numpy(off).cuda(), torch.from_numpy(by).cuda(), torch.from_numpy((1 - nulls).astype(np.uint8)).cuda()


def test_device_resident_input_through_the_c_abi():
    """offsets, bytes and validity as torch CUDA tensors (one DEVICE call), and device strings next to a host key column (MIXED)"""
    import torch
    from oracle import oracle as O
    from vaex_b200 import superagg
    rng = np.random.default_rng(5)
    n, ncat = 20_011, 37
    x = rng.integers(-1, ncat + 1, n).astype("i8")
    words = ["", "ab", "äß€ü", "q" * 100, "r" * 17]
    strs = [None if rng.random() < 0.1 else words[rng.integers(0, len(words))] for _ in range(n)]
    off, by, valid = _device_strings(strs)
    cells = O.flat_indices([O.ordinal(x, ncat, 0)], n)[0].astype(np.int64)
    for dropnull in (False, True):
        want = agg_list_string(cells, strs, ncat + 2, dropnull=dropnull)
        for key_on_device in (True, False):
            b = superagg.BinnerOrdinal_int64(1, "x", ncat, 0, False, False)
            g = superagg.Grid([b])
            a = superagg.AggList_string_int64(g, 1, 1, False, dropnull)
            b.set_data(0, torch.from_numpy(x).cuda() if key_on_device else x)
            a.set_buffers(0, off, by, valid)
            torch.cuda.synchronize()
            g.bin(0, [a], n)
            for gv, wv in zip(a.result_arrays(), want):
                assert np.array_equal(gv, wv), (dropnull, key_on_device)
    # a second call appends behind the first (arrival order = call order), device offsets that do not start at 0
    b = superagg.BinnerOrdinal_int64(1, "x", ncat, 0, False, False)
    g = superagg.Grid([b])
    a = superagg.AggList_string_int64(g, 1, 1)
    xd = torch.from_numpy(x).cuda()
    cut = 7_777
    for i1, i2 in ((0, cut), (cut, n)):
        b.set_data(0, xd[i1:i2])
        a.set_buffers(0, off[i1:i2 + 1], by, valid[i1:i2])
        torch.cuda.synchronize()
        g.bin(0, [a], i2 - i1)
    for gv, wv in zip(a.result_arrays(), agg_list_string(cells, strs, ncat + 2)):
        assert np.array_equal(gv, wv)


def test_sliced_arrow_input():
    import pyarrow as pa
    from oracle import oracle as O
    from vaex_b200 import superagg
    rng = np.random.default_rng(6)
    n = 5000
    strs = [None if rng.random() < 0.1 else "s%d" % rng.integers(0, 10 ** rng.integers(1, 9)) for _ in range(n)]
    x = rng.integers(0, 4, n).astype("i4")
    full = pa.array(strs, type=pa.large_string())
    part = full[137:4500]
    assert np.frombuffer(part.buffers()[1], np.int64, count=1, offset=part.offset * 8)[0] != 0
    b = superagg.BinnerOrdinal_int32(1, "x", 4, 0, False, False)
    g = superagg.Grid([b])
    a = superagg.AggList_string_int64(g, 1, 1)
    b.set_data(0, np.ascontiguousarray(x[137:4500]))
    a.set_data(0, part, 0)
    g.bin(0, [a], len(part))
    cells = O.flat_indices([O.ordinal(x[137:4500], 4, 0)], len(part))[0].astype(np.int64)
    for gv, wv in zip(a.result_arrays(), agg_list_string(cells, strs[137:4500], 6)):
        assert np.array_equal(gv, wv)
    assert a.get_result().to_pylist()[:4] == [[s for s, c in zip(strs[137:4500], x[137:4500]) if c == k] for k in range(4)]


def test_output_past_4gb():
    """4200 strings of 1,048,581 bytes (4.4e9 bytes in all, > 2^32) made on the device, in 3 groups: the string offsets and the
    gathered bytes past 2^32 are checked in full, which a 32-bit offset in the scan or the gather would break"""
    import torch
    from vaex_b200 import superagg
    count, width = 4200, 1_048_581  # width % 16 != 0: the strings start at every alignment
    rows = torch.arange(count, device="cuda")
    pattern = (torch.arange(width, device="cuda") % 256).to(torch.uint8)
    data = (pattern[None, :] + (rows % 256).to(torch.uint8)[:, None]).reshape(-1)  # byte p of string i = (p + i) % 256
    offsets = torch.arange(count + 1, device="cuda", dtype=torch.int64) * width
    keys = (rows % 3).to(torch.int64)
    b = superagg.BinnerOrdinal_int64(1, "k", 3, 0, False, False)
    g = superagg.Grid([b])
    a = superagg.AggList_string_int64(g, 1, 1)
    b.set_data(0, keys)
    a.set_buffers(0, offsets, data)
    torch.cuda.synchronize()
    g.bin(0, [a], count)
    lo, so, by, va = a.result_arrays()  # waits for the bin() call: only then may the input go
    del data
    torch.cuda.empty_cache()
    assert lo.tolist() == [0, 1400, 2800, 4200, 4200, 4200]
    assert so[-1] == count * width > 2 ** 32 and np.array_equal(so, np.arange(count + 1, dtype=np.int64) * width)
    assert va.all()
    order = np.concatenate([np.arange(c, count, 3) for c in range(3)])  # the strings of cell 0, then 1, then 2, each in row order
    base = (np.arange(width) % 256).astype(np.uint8)
    for k in range(0, count, 200):
        block = by[k * width:(k + 200) * width].reshape(-1, width)
        want = (base[None, :] + (order[k:k + 200] % 256).astype(np.uint8)[:, None]).astype(np.uint8)
        assert np.array_equal(block, want), k


def test_string_list_refuses_the_numeric_read_and_more_grids():
    from vaex_b200 import _lib, superagg
    g = superagg.Grid([superagg.BinnerOrdinal_int64(1, "k", 3)])
    with pytest.raises(RuntimeError, match="list aggregation only accepts 1 grid"):
        superagg.AggList_string_int64(g, 2, 1)
    a = superagg.AggList_string_int64(g, 1, 1)
    with pytest.raises(RuntimeError, match="b200_agg_list_string_read"):
        a._read()
    out = np.zeros(8, np.int64)
    assert _lib.lib().b200_agg_list_read(a._h, out.ctypes.data, None) != 0
    assert a.get_result().to_pylist() == [[]] * 5
    assert a.__sizeof__() == 0
