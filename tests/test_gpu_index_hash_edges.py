"""index_hash_<T> on the device at key edges (tests/index_hash_edge_cases.py): against the compiled reference's answers
(index_hash_edges_golden.npz) and against the restatement in bit-pattern mode, on host, page-locked and device inputs; the sentinel
key, NaN payloads, +-0.0, row spans at byte boundaries, table growth across a byte of the table size, and lookups with keys of
every other dtype."""
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
from test_gpu_index_hash import vector_duplicates  # noqa: E402

pytestmark = pytest.mark.gpu

PLACES = ["host", "pinned", "device"]
KEY_DTYPES = E.DTYPES + ["datetime64[ns]"]


def device_classes(dtype):
    from vaex_b200 import superutils
    return getattr(superutils, "index_hash_" + dtype)


def put(a, place):
    """a host array on the host, page-locked, or on the device (datetimes as a typed device view of their ticks)"""
    import torch
    if a is None or place == "host":
        return a
    a = np.ascontiguousarray(a)
    if place == "pinned":
        return torch.from_numpy(a.view(f"u{a.itemsize}")).pin_memory().numpy().view(a.dtype)
    if a.dtype.kind == "M":
        from vaex_b200.expression import DeviceArray
        t = torch.from_numpy(a.view(np.int64)).cuda()
        return DeviceArray(t.data_ptr(), len(a), a.dtype, keep=t)
    return torch.from_numpy(a).cuda()


def host(x):
    return np.asarray(x.cpu() if hasattr(x, "cpu") else x)


def drive(case, place):
    """the device index of a case: its updates, then each merged index"""
    def build(updates):
        h = device_classes(case["dtype"])(case["nmaps"])
        for keys, mask, start in updates:
            if mask is None:
                h.update(put(keys, place), start)
            else:
                h.update(put(keys, place), put(mask, place), start)
        return h
    h = build(case["updates"])
    for m in case["merges"]:
        h.merge(build(m))
    return h


def restate(case):
    def build(updates):
        o = IO.IndexHash(case["dtype"], case["nmaps"], bits=True)
        for keys, mask, start in updates:
            o.update(keys, mask, start)
        return o
    o = build(case["updates"])
    for m in case["merges"]:
        o.merge(build(m))
    return o


def results(h, case, place):
    """G.run's results of a built device index, its lookups placed like its keys"""
    import torch
    look, lmask = put(case["lookup"], place), put(case["lookup_mask"], place)
    res = {}
    res["map"] = host(h.map_index(look) if lmask is None else h.map_index_masked(look, lmask)).astype(np.int64)
    for w in G.WIDTHS:
        n = len(case["lookup"])
        o = torch.zeros(n, dtype=getattr(torch, w), device="cuda") if place == "device" else np.zeros(n, w)
        unknown = h.map_index(look, o) if lmask is None else h.map_index_masked(look, lmask, o)
        res["unknown_" + w], res["map_" + w] = np.array(bool(unknown)), host(o)
    left, right = h.map_index_duplicates(look, case["dup_start"])
    res["dup_left"], res["dup_right"] = host(left), host(right)
    res["scalars"] = np.array([len(h), h.count, h.has_duplicates, h.nan_count, h.null_count], np.int64)
    return res


def same(got, want, name):
    assert set(got) == set(want), name
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), f"{name}: {k}\n{np.asarray(got[k])}\n{np.asarray(want[k])}"


def check_shards(h, o, name):
    """extract() / offsets() against the restatement's union: every key once, with its primary row, in the shard of its hash"""
    keys, rows, shards = h._extract_arrays()
    c = S.canon(keys)
    assert len(set(c.tolist())) == len(c), name
    assert dict(zip(c.tolist(), rows.tolist())) == o.extract(), name
    assert np.array_equal(shards, S.shard_of(keys, h.nmaps)), name
    assert len(h.extract()) == h.nmaps, name
    sizes = np.bincount(shards, minlength=h.nmaps)
    sizes[0] += h.offset
    assert h.offsets() == [0] + np.cumsum(sizes)[:-1].tolist(), name


@pytest.mark.parametrize("place", PLACES)
def test_golden_vectors(place):
    golden = GE.load()
    assert len(golden) == len(GE.cases())
    for name, (case, res) in golden.items():
        h = drive(case, place)
        same(results(h, case, place), res, name)
        if place == "host":
            check_shards(h, restate(case), name)


@pytest.mark.parametrize("place", PLACES)
def test_sequential_every_nmaps_against_restatement(place):
    """every dtype x nmaps of the sequential cases (the golden file stores a rotation of them; the restatement is pinned on all of them
    against the compiled classes)"""
    for name, case in E.all_sequential(zeros=False).items():
        h = drive(case, place)
        same(results(h, case, place), G.run(lambda dt: IO.classes(dt, True), case), name)
        if place == "host":
            check_shards(h, restate(case), name)


@pytest.mark.parametrize("place", PLACES)
def test_unordered_against_restatement(place):
    for name, case in E.all_unordered(zeros=True).items():
        h = drive(case, place)
        same(results(h, case, place), G.run(lambda dt: IO.classes(dt, True), case), name)
        check_shards(h, restate(case), name)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_nan_payloads_share_one_row(dtype):
    nans = S.nan_values(dtype)
    for place in PLACES:
        h = device_classes(dtype)(3)
        keys = np.concatenate([np.ones(1, dtype), nans, np.full(1, 2, dtype)])  # the payloads' own bits, not a float64 round trip
        mask = np.zeros(len(keys), np.uint8)
        mask[-1] = 1
        h.update(put(keys, place), put(mask, place), 40)
        assert (h.nan_count, h.null_count, h.count) == (len(nans), 1, 3)
        assert host(h.map_index(put(nans, place))).tolist() == [40 + len(nans)] * len(nans)
        # a masked NaN is still the NaN row (NaN comes first, as in the reference), the null row only for masked numbers
        got = h.map_index_masked(put(np.array([nans[2], 2.0, 1.0], dtype), place), put(np.array([1, 1, 0], np.uint8), place))
        assert host(got).tolist() == [40 + len(nans), 41 + len(nans), 40]


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_signed_zeros_are_two_keys(dtype):
    """the documented deviation: keys compare by bit pattern, so -0.0 and 0.0 are two keys with two rows"""
    for place in PLACES:
        h = device_classes(dtype)(1)
        h.update(put(np.array([0.0, 5.0, -0.0], dtype), place), 0)
        assert host(h.map_index(put(np.array([0.0, -0.0], dtype), place))).tolist() == [0, 2]
        assert h.count == 3 and not h.has_duplicates


def test_table_grows_across_a_byte_between_update_and_duplicates():
    """duplicates are read (rows sorted into per-slot ranges for a 2^16-slot table), then the table grows to 2^17 slots: the sentinel's
    range moves from seg[2^16] to seg[2^17], and slot numbers need a third byte"""
    import torch
    rng = np.random.default_rng(17)
    for dtype in ("int64", "uint64", "int32"):
        s = S.sentinel(dtype)
        # one call of 30000 rows sizes the table to 2^16 slots, the next one of 40000 to 2^17 (twice the rows the call could add)
        k1 = rng.integers(1, 15_000, 30_000).astype(dtype)
        k1[[3, 9_000, 29_999]] = s
        k2 = rng.integers(1, 60_000, 40_000).astype(dtype)
        k2[[0, 37_777]] = s
        look = np.concatenate([rng.integers(0, 62_000, 20_000).astype(dtype), np.array([s, s], dtype)])
        h, o = device_classes(dtype)(7), IO.IndexHash(dtype, 7, bits=True)
        h.update(torch.from_numpy(k1).cuda(), 100)
        o.update(k1, None, 100)
        size1 = h.__sizeof__()
        left, right = h.map_index_duplicates(look, 0)
        wl, wr = vector_duplicates(k1, look, 0)
        assert np.array_equal(left, wl) and np.array_equal(right, wr + 100)
        h.update(k2, -len(k2))
        o.update(k2, None, -len(k2))
        assert h.__sizeof__() > size1
        both = np.concatenate([k2, k1])  # rows -len(k2) .. -1, then a gap to 100 ..
        rows = np.concatenate([np.arange(-len(k2), 0), 100 + np.arange(len(k1))])
        left, right = h.map_index_duplicates(torch.from_numpy(look).cuda(), 5, device=True)
        wl, wr = vector_duplicates(both, look, 5)
        assert np.array_equal(left.cpu().numpy(), wl) and np.array_equal(right.cpu().numpy(), rows[wr])
        got = host(h.map_index(look))
        want, _ = IO.IndexHash.map_index(o, look)
        assert np.array_equal(got, want) and got[-1] == -len(k2)
        assert (len(h), h.count, h.has_duplicates) == (len(o), o.count, o.has_duplicates)


def test_row_span_bytes_with_long_overflows():
    """one key whose rows straddle every row-byte boundary up to 2^24: its overflow must come back in row order"""
    rows = np.array(sorted({0, 1, 254, 255, 256, 257, 65534, 65535, 65536, 65537, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1}))
    for dtype in ("int64", "uint64", "int8"):
        s = S.sentinel(dtype)
        for key in (np.array([7], dtype)[0], s):
            h = device_classes(dtype)(3)
            for r in rows[::-1]:  # one call per row, newest first
                h.update(np.array([key, 3], dtype), int(r) - 5)
            left, right = h.map_index_duplicates(np.array([key], dtype), 0)
            assert host(h.map_index(np.array([key], dtype))).tolist() == [rows[0] - 5]
            assert host(right).tolist() == (rows[1:] - 5).tolist() and host(left).tolist() == [0] * (len(rows) - 1)
            left, right = h.map_index_duplicates(np.array([3], dtype), 0)
            assert host(right).tolist() == (rows[1:] - 4).tolist()


def _matrix_index(idx_dtype, key_dtype):
    """an index of `idx_dtype` holding the key dtype's edge values cast by value, plus its own edge values; the keys to look up"""
    kdt = np.dtype(key_dtype)
    if kdt.kind == "M":
        keys = S.edge_values("int64").view(kdt)
    else:
        keys = np.concatenate([S.edge_values(kdt), S.nan_values(kdt)]).astype(kdt)
    with np.errstate(invalid="ignore", over="ignore"):
        cast = (keys.view(np.int64) if kdt.kind == "M" else keys).astype(idx_dtype)
    content = np.concatenate([S.edge_values(idx_dtype), cast[::-1]]).astype(idx_dtype)
    return content, keys


@pytest.mark.parametrize("idx_dtype", E.DTYPES)
def test_lookup_keys_of_every_dtype(idx_dtype):
    """a key column of another dtype is cast by value where numpy calls the cast safe, whatever its placement, and refused with the
    same TypeError everywhere else: a device column is never read by its bits as a different type"""
    for key_dtype in KEY_DTYPES:
        content, keys = _matrix_index(idx_dtype, key_dtype)
        h = device_classes(idx_dtype)(3)
        h.update(content, 0)
        o = IO.IndexHash(idx_dtype, 3, bits=True)
        o.update(content, None, 0)
        mask = (np.arange(len(keys)) % 5 == 1).astype(np.uint8)
        for place in PLACES:
            what = f"{key_dtype} keys on index_hash_{idx_dtype}, {place}"
            if np.can_cast(keys.dtype, idx_dtype, "safe"):
                want, _ = IO.IndexHash.map_index(o, keys)
                assert np.array_equal(host(h.map_index(put(keys, place))), want), what
                want, _ = IO.IndexHash.map_index(o, keys, mask)
                assert np.array_equal(host(h.map_index_masked(put(keys, place), put(mask, place))), want), what
                left, right = h.map_index_duplicates(put(keys, place), 3)
                wl, wr = IO.IndexHash.map_index_duplicates(o, keys, 3)
                assert np.array_equal(host(left), wl) and np.array_equal(host(right), wr), what
            else:
                with pytest.raises(TypeError, match="incompatible key dtype"):
                    h.map_index(put(keys, place))
                with pytest.raises(TypeError, match="incompatible key dtype"):
                    h.map_index_masked(put(keys, place), put(mask, place))
                with pytest.raises(TypeError, match="incompatible key dtype"):
                    h.map_index_duplicates(put(keys, place), 0)
