"""The row movers at the edges of the code they share: the argsort of Frame.sort across radix blocks (radix.cuh: 4096 rows per
block up to 2048 blocks, then the tile doubles) and at the 16-key packing limit; b200_take over every fixed-width dtype, source kind
and the 16-column launch split; the string gathers (copy_string of strings.cuh) at every source and destination alignment and at
each group width; and the numeric AggList where its sort key cell * 4 + category crosses a byte.

References: sort_oracle (pinned to pa.compute.sort_indices) and row_movers_oracle (pinned to sort_oracle and oracle.agg_list by
test_row_movers_oracle_cpu.py), numpy fancy indexing and Python slicing; values are compared bit for bit."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [HERE, os.path.dirname(HERE)]
import row_movers_oracle as R  # noqa: E402
import sort_oracle as S  # noqa: E402

pytestmark = pytest.mark.gpu

KINDS = S.NUMERIC + S.TIMES + ["string"]


def bits(a):
    """the values of a numpy array as native unsigned integers of their width (NaN payloads, -0.0 and byte order kept apart)"""
    a = np.asarray(a)
    isz = a.dtype.itemsize
    order = a.dtype.byteorder if a.dtype.byteorder in "<>" else "="
    return a.view(np.dtype(f"u{isz}").newbyteorder(order)).astype(f"=u{isz}")


def host(x):
    """a result column (torch tensor, numpy or np.ma) as (numpy data, numpy bool mask or None)"""
    if hasattr(x, "__cuda_array_interface__") and not isinstance(x, np.ndarray):
        import torch
        from vaex_b200 import _lib
        _lib.context().sync()
        x = torch.as_tensor(x, device="cuda").cpu().numpy()
    if np.ma.isMaskedArray(x):
        return np.asarray(x.data), np.ma.getmaskarray(x)
    return np.asarray(x), None


# ---- 1. the argsort across radix blocks -------------------------------------------------------------------------------------------
def corpus_key(rng, kind, n, masked, byteswap, descending):
    if kind == "string":
        return R.string_key(rng, n, masked, descending)
    return S.random_key(rng, kind, n, masked, byteswap, descending)


def key_frame(keys, on_device=False, extra=None, filter=None):
    """a frame with the keys as columns k0..: strings as arrow, masked keys as np.ma, plain native numeric ones on the device when
    `on_device`"""
    import torch
    from vaex_b200.frame import Frame
    columns = {}
    for i, (v, m, *_) in enumerate(keys):
        if v.dtype.kind == "O":
            columns[f"k{i}"] = R.arrow_strings(keys[i])
        elif m is not None:
            columns[f"k{i}"] = np.ma.array(v, mask=m)
        elif on_device and v.dtype.kind in "biuf" and v.dtype.isnative:
            columns[f"k{i}"] = torch.from_numpy(v).cuda()
        else:
            columns[f"k{i}"] = v
    columns.update(extra or {})
    return Frame(columns, filter=filter)


def device_order(keys, on_device=False, extra=None, filter=None):
    """the unfiltered row numbers in the order df.sort puts them (sort.sorted_rows: staging, compaction, b200_argsort)"""
    from vaex_b200 import sort as _sort
    df = key_frame(keys, on_device, extra, filter)
    rows = _sort.sorted_rows(df, [f"k{i}" for i in range(len(keys))], [not k[2] for k in keys])
    return rows.cpu().numpy()


def check_sort(keys, on_device=False, arrow=False):
    got, want = device_order(keys, on_device), R.argsort(keys)
    bad = np.flatnonzero(got != want)
    assert not len(bad), (len(bad), bad[:5], got[bad[:5]], want[bad[:5]])
    if arrow:
        assert np.array_equal(want, S.arrow_argsort([k[:3] for k in keys]))


SMALL = [4095, 4096, 4097, 2 * 4096 + 1]                  # one radix block, a full one, one row and one block past it
LARGE = [8_388_607, 8_388_608, 8_388_609, 2 ** 24 + 3]    # both sides of the 2048-block cap where the tile doubles, and past it


@pytest.mark.parametrize("n", SMALL)
def test_argsort_block_edges(n):
    """every kind masked / byte-swapped / descending alone, then 2-4 mixed keys, against numpy and arrow"""
    rng = np.random.default_rng(n)
    for kind in KINDS:
        for flags in range(8):
            check_sort([corpus_key(rng, kind, n, bool(flags & 1), bool(flags & 2), bool(flags & 4))], on_device=flags == 0, arrow=True)
    for nkeys in (2, 3, 4):
        for trial in range(4):
            keys = [corpus_key(rng, rng.choice(KINDS), n, rng.random() < 0.4, rng.random() < 0.3, rng.random() < 0.5) for _ in range(nkeys)]
            check_sort(keys, on_device=trial % 2 == 1, arrow=True)


@pytest.mark.parametrize("n", LARGE)
def test_argsort_many_blocks(n):
    """1, 2, 3 and 4 keys at sizes past one radix block; the 14 kinds rotate over the sizes so each one sorts there"""
    j = LARGE.index(n)
    rng = np.random.default_rng(n)
    slot = 10 * j
    for nkeys in (1, 2, 3, 4):
        keys = []
        for s in range(slot, slot + nkeys):
            keys.append(corpus_key(rng, KINDS[s % len(KINDS)], n, s % 2 == 1, s % 3 == 0, s % 5 in (1, 3)))
        slot += nkeys
        check_sort(keys, on_device=(nkeys + j) % 2 == 1)


def test_argsort_stable_across_blocks():
    """half the rows share the first key's value, the second key has two values: the order of the ties, which cross every radix
    block, is the row order"""
    n = 8_388_609
    rng = np.random.default_rng(7)
    first = S.random_key(rng, "float64", n, True, False, False)
    values = first[0].copy()
    values[rng.random(n) < 0.5] = 1.5
    first = (values, first[1], False)
    check_sort([first])
    check_sort([(values, first[1], True), (rng.random(n) < 0.5, None, False)])


# ---- 2. key packing -----------------------------------------------------------------------------------------------------------
def narrow_key(rng, kind, n, masked, byteswap, descending, nan=False):
    """a corpus key over three of its kind's edge values (always a NaN / NaT with `nan`), so that every one of 16 keys decides ties"""
    if kind == "string":
        key = R.string_key(rng, n, masked, descending)
        codes = rng.choice(len(S.STRINGS), 3, replace=False)[rng.integers(0, 3, n)]
        return S.STRINGS[codes], key[1], descending, codes
    ev = S.edge_values(kind)
    k = min(3, len(ev))
    pick = list(rng.choice(len(ev), k, replace=False))
    if nan:
        pick[0] = len(ev) - 1 if ev.dtype.kind == "f" else 3  # a NaN payload / NaT (INT64_MIN)
    values = ev[np.array(pick)[rng.integers(0, k, n)]]
    if byteswap and values.dtype.itemsize > 1:
        values = values.astype(values.dtype.newbyteorder("S"))
    return values, (rng.random(n) < 0.2) if masked else None, descending


# (kind, masked, byte-swapped, descending, NaN / NaT drawn): f64 with both class bits, NaT-as-null datetimes, strings, masked i32...
SIXTEEN = [("float64", True, False, False, True), ("int8", False, True, True, False), ("bool", False, False, False, False),
           ("int32", True, False, True, False), ("datetime64[ns]", False, True, False, True), ("string", False, False, False, False),
           ("float64", True, True, True, True), ("float32", False, True, False, True), ("uint16", True, False, False, False),
           ("int64", True, True, True, False), ("bool", True, False, True, False), ("timedelta64[s]", False, False, True, True),
           ("float64", True, False, True, True), ("uint8", False, False, False, False), ("string", True, False, True, False),
           ("int16", False, True, False, False)]


def test_sixteen_keys_straddle_words():
    rng = np.random.default_rng(16)
    n = 100_000
    keys = [narrow_key(rng, kind, n, masked, swap, desc, nan) for kind, masked, swap, desc, nan in SIXTEEN]
    check_sort(keys, arrow=True)
    check_sort(keys[::-1], on_device=True, arrow=True)


def packing_cases():
    """name -> (keys, k_sort_encode launches (words), k_radix_scatter launches or None)"""
    rng = np.random.default_rng(32)
    n = 100_000
    const = [(np.full(n, 1000 + i, "i8"), None, i % 2 == 1) for i in range(16)]
    varying = list(const)
    varying[7] = (rng.integers(0, 256, n).astype("i8"), None, False)  # one byte of one word varies: one pass in 16 rounds
    class_only = const[:15] + [(np.zeros(n, "u1"), rng.random(n) < 0.3, False)]  # value 0 in every row, null or not
    return {
        "16 masked float64": ([narrow_key(rng, "float64", n, True, i % 3 == 0, i % 2 == 1, True) for i in range(16)], 32, None),
        "one varying word": (varying, 16, 1),
        "only the class field varies": (class_only, 16, 1),
    }


def _record_packing():
    """the encode / scatter launches of every packing case, in a fresh process (see test_gpu_sort._record_paths)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, (keys, _, _) in packing_cases().items():
        device_order(keys)  # warm-up
        for attempt in range(10):  # a session now and then comes back without kernel records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                got = device_order(keys)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
            if names:
                break
        out[name] = {"encode": sum("k_sort_encode" in x for x in names), "scatter": sum("k_radix_scatter" in x for x in names),
                     "correct": bool(np.array_equal(got, R.argsort(keys))), "kernels": len(names)}
    return out


def _record_gathers():
    """the k_take_str_copy widths every string gather case launched"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, (arr, index, _) in string_cases().items():
        if not profiled(name):
            continue
        for attempt in range(10):  # a session now and then comes back without kernel records
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                got = gathered(arr, index)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
            if names:
                break
        out[name] = {"widths": sorted({int(w) for x in names for w in re.findall(r"k_take_str_copy<(\d+)>", x)}),
                     "correct": got == expected_strings(arr, index), "kernels": len(names)}
    return out


@pytest.fixture(scope="module")
def recorded(tmp_path_factory):
    """the kernels the packing and string cases launched, recorded with torch.profiler in a process of its own"""
    out = tmp_path_factory.mktemp("prof") / "row_movers.json"
    subprocess.check_call([sys.executable, os.path.abspath(__file__), str(out)], cwd=os.path.dirname(HERE))
    return json.loads(out.read_text())


@pytest.mark.parametrize("name", sorted(packing_cases()))
def test_packing_rounds(recorded, name):
    keys, words, passes = packing_cases()[name]
    got = recorded["packing"][name]
    assert got["kernels"] > 0, "torch.profiler recorded no CUDA kernel"
    assert got["correct"], name
    assert got["encode"] == words, got
    if passes is not None:
        assert got["scatter"] == passes, got
    check_sort(keys)


def test_seventeen_keys_refused():
    from vaex_b200.frame import Frame
    df = Frame({f"k{i}": np.arange(10) for i in range(17)})
    with pytest.raises(ValueError, match="between 1 and 16 keys are supported, got 17"):
        df.sort([f"k{i}" for i in range(17)])


def test_filtered_sixteen_masked_keys(monkeypatch):
    """a filtered sort compacts the row numbers, 16 keys and their 16 masks: 33 columns in calls of 16, 16 and 1"""
    from vaex_b200 import expression as _expr
    calls = []
    compact = _expr.compact

    def counted(slot, keep, columns):
        calls.append(len(columns))
        return compact(slot, keep, columns)
    monkeypatch.setattr(_expr, "compact", counted)
    rng = np.random.default_rng(33)
    n = 100_000
    keys = [narrow_key(rng, kind if kind != "string" else "uint32", n, True, swap, desc, nan)
            for kind, _, swap, desc, nan in SIXTEEN]
    keep = rng.random(n) < 0.6
    got = device_order(keys, extra={"f": keep.astype("i1")}, filter="f > 0")
    assert calls == [16, 16, 1]
    kept = np.flatnonzero(keep)
    want = kept[R.argsort([(v[keep], m[keep], d) for v, m, d in keys])]
    assert np.array_equal(got, want)


# ---- 3. b200_take over every dtype ---------------------------------------------------------------------------------------------
TAKE_DTYPES = S.NUMERIC + ["datetime64[ns]", "timedelta64[s]"]
EXTRA = {"host": ["float32", "float64", "uint64", "int8", "bool", "datetime64[ns]", "timedelta64[s]"],
         "device": ["float32", "float64", "uint64", "int8", "bool", "uint16", "datetime64[ns]"]}


def take_source(rng, dtype, n):
    """random bits of the dtype, with its edge values (NaN payloads, -0.0, u8 >= 2^63, NaT, ...) planted, one in the last row"""
    dt = np.dtype(dtype)
    if dt.kind == "b":
        v = rng.random(n) < 0.5
    else:
        v = rng.integers(0, 256, n * dt.itemsize, dtype=np.uint8).view(dt).copy()
    ev = S.edge_values(dtype)
    v[rng.choice(n - 1, len(ev), replace=False)] = ev
    v[-1] = ev[-1]
    return v


def take_columns(source, n, seed):
    """20 columns of one source kind: name -> (column as the frame holds it, host values, mask or None)"""
    import torch
    rng = np.random.default_rng(seed)
    dtypes = TAKE_DTYPES + EXTRA["device" if source == "device" else "host"]
    assert len(dtypes) == 20
    out = {}
    for i, dtype in enumerate(dtypes):
        v = take_source(rng, dtype, n)
        mask = None
        col = v
        if source == "bigendian" and v.dtype.itemsize > 1:
            v = col = v.astype(v.dtype.newbyteorder(">"))
        elif source == "masked":
            mask = rng.random(n) < 0.3
            col = np.ma.array(v, mask=mask)
        elif source == "device" and v.dtype.kind in "mM":
            from vaex_b200.expression import DeviceArray
            t = torch.from_numpy(v.view("i8")).cuda()
            col = DeviceArray(t.data_ptr(), n, v.dtype, keep=t)  # torch has no datetime dtype
        elif source == "device":
            col = torch.from_numpy(v).cuda()
        out[f"c{i}_{dtype}"] = (col, v, mask)
    return out


@pytest.mark.parametrize("source", ["host", "bigendian", "masked", "device"])
def test_take_every_dtype(source):
    import torch
    from vaex_b200 import _lib
    from vaex_b200 import join as _join
    from vaex_b200.frame import Frame
    n = 50_001
    cols = take_columns(source, n, ["host", "bigendian", "masked", "device"].index(source))
    rng = np.random.default_rng(99)
    idx = rng.integers(-1, n, 30_000)
    idx[:4] = [n - 1, -1, 0, n - 1]
    # join.take: 20 columns in launches of 16 and 4, a missing row (-1) and the last row, host and device outputs
    for index in (idx, torch.from_numpy(idx.astype("i4")).cuda()):
        for device in (False, True):
            res = _join.take(index, [(_lib.split_mask(c)[0], m) for c, _, m in cols.values()], n, device)
            for (name, (_, v, m)), (values, valid) in zip(cols.items(), res):
                got, _ = host(values)
                want = np.where(idx >= 0, bits(v)[idx], 0)
                assert np.array_equal(bits(got), want), (name, device)
                valid = host(valid)[0]
                want_valid = (idx >= 0) & (True if m is None else ~m[idx])
                assert np.array_equal(valid.astype(bool), want_valid), name
    # Frame.take: every column's values and mask, placement kept (device datetimes come back to the host: torch has no such dtype)
    rows = idx.copy()
    rows[rows < 0] = n - 1
    out = Frame({name: c for name, (c, _, _) in cols.items()}).take(rows)
    for name, (c, v, m) in cols.items():
        got, got_mask = host(out.columns[name])
        assert np.array_equal(bits(got), bits(v)[rows]), name
        assert _lib.is_device(out.columns[name]) == (source == "device" and v.dtype.kind not in "mM"), name
        if m is not None:
            assert np.array_equal(got_mask, m[rows]), name


# ---- 4. string gathers at every alignment ---------------------------------------------------------------------------------------
LENGTHS = [0, 1, 15, 16, 17, 31, 33, 255, 257, 4099]
NULL_ROWS = 8


def aligned_source(seed, large, sliced):
    """(arrow string array, target rows {(length, start mod 16): row}): rows 0..15 are pads of length 0..15, then NULL_ROWS null rows
    over non-empty slots, then every length of LENGTHS starting at every offset mod 16 of the buffer; a sliced array drops a prefix"""
    import pyarrow as pa
    rng = np.random.default_rng(seed)
    lengths, valid, targets = [], [], {}
    prefix = [5, 9, 3] if sliced else []
    lengths += prefix + list(range(16))
    valid += [True] * len(lengths)
    lengths += [5 + 7 * i for i in range(NULL_ROWS)]
    valid += [False] * NULL_ROWS
    pos = sum(lengths)
    for L in LENGTHS:
        for s in range(16):
            gap = (s - pos) % 16
            if gap:
                lengths.append(gap)
                valid.append(True)
                pos += gap
            targets[(L, s)] = len(lengths) - len(prefix)
            lengths.append(L)
            valid.append(True)
            pos += L
    offsets = np.zeros(len(lengths) + 1, np.int64)
    offsets[1:] = np.cumsum(lengths)
    data = rng.integers(0, 256, int(offsets[-1]), dtype=np.uint8)
    bitmap = pa.py_buffer(np.packbits(np.array(valid), bitorder="little"))
    cls, odt = (pa.LargeStringArray, np.int64) if large else (pa.StringArray, np.int32)
    arr = cls.from_buffers(len(lengths), pa.py_buffer(offsets.astype(odt)), pa.py_buffer(data), bitmap, valid.count(False))
    return arr.slice(len(prefix)), targets


def source_strings(arr):
    """the rows of an arrow string array as bytes (None = null), from its buffers"""
    import pyarrow as pa
    isz = 8 if pa.types.is_large_string(arr.type) else 4
    off = np.frombuffer(arr.buffers()[1], np.int64 if isz == 8 else np.int32, count=len(arr) + 1, offset=arr.offset * isz)
    data = np.frombuffer(arr.buffers()[2], np.uint8)
    valid = arr.is_valid().to_numpy(zero_copy_only=False)
    return [data[off[i]:off[i + 1]].tobytes() if valid[i] else None for i in range(len(arr))]


def expected_strings(arr, index):
    src = source_strings(arr)
    return [src[i] if i >= 0 else None for i in index]


def gathered(arr, index):
    from vaex_b200 import join as _join
    out, _ = _join.take_strings(np.asarray(index), arr)
    return source_strings(out)


def width_for(mean):
    """the group width b200_take_strings picks for a mean string length"""
    return 32 if mean > 256 else 8 if mean > 32 else 4


def alignment_index(arr, targets, width):
    """every target gathered to every destination offset mod 16 (a pad of the right length before it), then the null rows and
    misses, then pads or long targets until the mean length selects `width`"""
    lengths = [0 if s is None else len(s) for s in source_strings(arr)]
    index, pos = [], 0
    for row in targets.values():
        for d in range(16):
            pad = (d - pos) % 16
            index += [pad, row]
            pos += pad + lengths[row]
    index += list(range(16, 16 + NULL_ROWS)) + [-1, -1]
    fill = 1 if width < width_for(pos // len(index)) else targets[(4099, 0)]
    while width_for(pos // len(index)) != width:
        index += [fill] * 64
        pos += 64 * lengths[fill]
    return np.array(index, np.int64)


def string_cases():
    """name -> (source, index, the group width its mean length selects)"""
    cases = {}
    for large in (False, True):
        for sliced in (False, True):
            arr, targets = aligned_source(40 + 2 * large + sliced, large, sliced)
            for width in (4, 8, 32):
                index = alignment_index(arr, targets, width)
                cases[f"{'int64' if large else 'int32'} offsets{' sliced' if sliced else ''} G={width}"] = (arr, index, width)
            # the buffer's last string alone, for every start offset mod 16 and a length of each width
            last = max(targets.values())
            for L, width in ((17, 4), (33, 8), (4099, 32)):
                for s in range(16):
                    sub = arr.slice(0, targets[(L, s)] + 1)
                    cases[f"{'int64' if large else 'int32'} offsets{' sliced' if sliced else ''} last L={L} s={s}"] = (sub, np.array([len(sub) - 1]), width)
            assert last == len(arr) - 1
    return cases


@pytest.mark.parametrize("large", [False, True])
@pytest.mark.parametrize("sliced", [False, True])
def test_string_gather_alignments(large, sliced):
    prefix = f"{'int64' if large else 'int32'} offsets{' sliced' if sliced else ''} "
    for name, (arr, index, width) in string_cases().items():
        if name.startswith(prefix) and (sliced or "sliced" not in name):
            got, want = gathered(arr, index), expected_strings(arr, index)
            bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
            assert not bad, (name, bad[:5])


def profiled(name):
    """the string cases whose kernels are recorded: every full alignment sweep, the last string alone at one offset per width"""
    return "last" not in name or name.endswith("s=15")


def test_string_gather_widths(recorded):
    """every case ran the k_take_str_copy width its mean length selects; all three ran"""
    seen = set()
    for name, (_, _, width) in string_cases().items():
        if not profiled(name):
            continue
        got = recorded["strings"][name]
        assert got["kernels"] > 0, "torch.profiler recorded no CUDA kernel"
        assert got["correct"], name
        assert got["widths"] == [width], (name, got)
        seen.add(width)
    assert seen == {4, 8, 32}


def list_string_layout(rng):
    """(strings, cell per string): every length of LENGTHS at every (pool offset, output offset) pair mod 16.  The targets go to
    cell 0, each after a cell-0 pad that puts its output offset (the cell-0 bytes before it) at the wanted residue and a cell-1 pad
    that puts its pool offset (all the bytes before it) at the wanted residue; cell 1 also holds null rows"""
    chars = "".join(chr(c) for c in rng.integers(33, 127, 8192))
    strs, cells, pool, out = [], [], 0, 0

    def put(length, cell):
        nonlocal pool, out
        at = int(rng.integers(0, len(chars) - length))
        strs.append(chars[at:at + length])
        cells.append(cell)
        pool += length
        out += length if cell == 0 else 0
    for L in LENGTHS:
        for src in range(16):
            for dst in range(16):
                put((dst - out) % 16, 0)
                put((src - pool) % 16, 1)
                if (src + dst) % 37 == 0:
                    strs.append(None)
                    cells.append(1)
                put(L, 0)
    return strs, np.array(cells, np.int64)


def test_agg_list_string_alignments():
    """every length of LENGTHS copied from every pool offset to every output offset mod 16 through AggList_string (its copy is
    copy_string too), the rows fed in three bin() calls"""
    import pyarrow as pa
    from oracle import oracle as O
    from oracle.agglist_string import agg_list_string
    from vaex_b200 import superagg
    strs, x = list_string_layout(np.random.default_rng(77))
    n, ncat = len(strs), 2
    lengths = np.array([0 if s is None else len(s) for s in strs])
    pool = np.concatenate([[0], np.cumsum(lengths)])[:-1]
    out = np.concatenate([[0], np.cumsum(np.where(x == 0, lengths, 0))])[:-1]
    covered = {(L, p % 16, o % 16) for L, p, o, c in zip(lengths, pool, out, x) if c == 0 and L in LENGTHS}
    assert len(covered) == len(LENGTHS) * 256
    cells = O.flat_indices([O.ordinal(x, ncat, 0)], n)[0].astype(np.int64)
    b = superagg.BinnerOrdinal_int64(1, "x", ncat, 0, False, False)
    g = superagg.Grid([b])
    a = superagg.AggList_string_int64(g, 1, 1)
    full = pa.array(strs, type=pa.large_string())
    for i1, i2 in ((0, 7), (7, 1001), (1001, n)):
        b.set_data(0, np.ascontiguousarray(x[i1:i2]))
        a.set_data(0, full[i1:i2], 0)
        g.bin(0, [a], i2 - i1)
    for gv, wv in zip(a.result_arrays(), agg_list_string(cells, strs, ncat + 2)):
        assert np.array_equal(gv, wv)


# ---- 5. numeric AggList where cell * 4 + category crosses a byte -----------------------------------------------------------------
# cells (ordinal bins + 2: the last two are the overflow cell, count, and the missing cell, count + 1, which an integer binner
# without a mask never fills) -> the byte bound the value records' keys cross.  The overflow cell holds the largest real key,
# 4 * (cells - 2) + category: at 66, 16,386 and 4,194,306 cells its value records' key is 256, 65,536 and 2^24; at 64 and 16,384
# cells only the skip key, cells * 4, crosses 255 and 65,535.
LIST_CELLS = {64: None, 66: 255, 16_384: None, 16_386: 65_535, 4_194_306: 2 ** 24 - 1}
CALL_LENGTHS = [1, 3, 1023, 1025, 70_001]
LIST_DTYPES = S.NUMERIC + [">f8", ">i4"]


def list_rows(rng, dtype, n, ncat):
    """ordinal keys in [-1, ncat] crowded at both ends (ncat: the overflow cell, the grid's last filled one), values of random bits
    with NaN payloads and -0.0 planted"""
    x = rng.integers(-1, ncat + 1, n)
    ends = rng.random(n)
    x[ends < 0.3] = ncat - rng.integers(0, 3, (ends < 0.3).sum())
    x[ends > 0.9] = rng.integers(-1, 2, (ends > 0.9).sum())
    dt = np.dtype(dtype)
    if dt.kind == "b":
        v = rng.random(n) < 0.5
    else:
        v = rng.integers(0, 256, n * dt.itemsize, dtype=np.uint8).view(dt).copy()
        if dt.kind == "f":
            ev = S.edge_values(dt.newbyteorder("=")).astype(dt)
            planted = rng.random(n) < 0.2
            v[planted] = ev[rng.integers(0, len(ev), planted.sum())]
    return x.astype("i8"), v


@pytest.mark.parametrize("dtype", LIST_DTYPES)
def test_agg_list_key_bytes(dtype):
    from oracle import oracle as O
    from vaex_b200 import superagg
    rng = np.random.default_rng(LIST_DTYPES.index(dtype))
    n = sum(CALL_LENGTHS)
    bounds = np.concatenate([[0], np.cumsum(CALL_LENGTHS)])
    calls = list(zip(bounds[:-1], bounds[1:]))
    dt = np.dtype(dtype)
    name = f"AggList_{dt.newbyteorder('=').name}_int64" + ("" if dt.isnative else "_non_native")
    for cells_n, bound in LIST_CELLS.items():
        ncat = cells_n - 2
        x, v = list_rows(rng, dtype, n, ncat)
        cells = O.flat_indices([O.ordinal(x, ncat, 0)], n)[0].astype(np.int64)
        assert cells.max() == ncat and (bound is None or 4 * ncat > bound)
        for masked in (False, True):
            valid = (rng.random(n) > 0.25).astype(np.uint8) if masked else None
            for dropnan in (False, True):
                for dropnull in (False, True):
                    b = superagg.BinnerOrdinal_int64(1, "x", ncat, 0, False, False)
                    g = superagg.Grid([b])
                    assert len(g) == cells_n
                    a = getattr(superagg, name)(g, 1, 1, dropnan, dropnull)
                    for i1, i2 in calls:
                        b.set_data(0, np.ascontiguousarray(x[i1:i2]))
                        a.set_data(0, np.ascontiguousarray(v[i1:i2]), 0)
                        if masked:
                            a.set_data_mask(0, np.ascontiguousarray(valid[i1:i2]))
                        g.bin(0, [a], i2 - i1)
                    offsets, values = a.result_arrays()
                    want_off, want, nulls = R.agg_list(cells, v, valid, cells_n, dropnan, dropnull, calls)
                    case = (cells_n, masked, dropnan, dropnull)
                    assert np.array_equal(offsets, want_off), case
                    assert values.dtype == want.dtype, case
                    assert np.array_equal(bits(values)[~nulls], bits(want)[~nulls]), case


if __name__ == "__main__":  # the profiling half of test_packing_rounds and test_string_gather_widths, in a process of its own
    result = {"packing": _record_packing(), "strings": _record_gathers()}
    with open(sys.argv[1], "w") as f:
        json.dump(result, f)
