"""GPU parity of index_hash_<dtype> (vaex_b200.superutils) against the golden vectors of the compiled reference, the sequential
restatement (tests/index_hash_oracle.py) and the compiled classes themselves where oracle/_ref exists."""
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import index_hash_oracle as IO  # noqa: E402
import make_golden_index_hash as G  # noqa: E402

pytestmark = pytest.mark.gpu


def device_classes(dtype):
    from vaex_b200 import superutils
    return getattr(superutils, "index_hash_" + dtype)


def same(got, want, name):
    for k in want:
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), f"{name}: {k}"


def test_golden_vectors():
    for name, (case, res) in G.load(os.path.join(HERE, "golden", "index_hash_golden.npz")).items():
        same(G.run(device_classes, case), res, name)


def test_against_compiled_reference(ref):
    su = ref.modules()[1]
    for name, case in G.cases().items():
        if case["nmaps"] == 3:
            same(G.run(device_classes, case), G.run(lambda dt: getattr(su, "index_hash_" + dt), case), name)


def state(h, look, lmask=None, start=0):
    rows = h.map_index_masked(look, lmask) if lmask is not None else h.map_index(look)
    left, right = h.map_index_duplicates(look, start)
    rows, left, right = (np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in (rows, left, right))
    return dict(rows=rows, left=left, right=right, scalars=np.array([len(h), h.count, h.has_duplicates, h.nan_count, h.null_count]))


def oracle_state(o, look, lmask=None, start=0):
    rows, _ = IO.IndexHash.map_index(o, look, lmask)
    left, right = IO.IndexHash.map_index_duplicates(o, look, start)
    return dict(rows=rows, left=left, right=right, scalars=np.array([len(o), o.count, o.has_duplicates, o.nan_count, o.null_count]))


def keys_of(rng, dtype, n, distinct):
    k = G._keys(rng, dtype, n, distinct)
    if k.dtype.kind == "f":
        k[rng.random(n) < 0.03] = np.nan
    return k


@pytest.mark.parametrize("dtype", G.DTYPES)
@pytest.mark.parametrize("nmaps", [1, 3, 7])
@pytest.mark.parametrize("place", ["host", "device", "pinned"])
def test_chunks_out_of_order_with_masks(dtype, nmaps, place):
    import torch
    rng = np.random.default_rng(zlib.crc32(f"{dtype} {nmaps} {place}".encode()))
    n = 20_000
    keys = keys_of(rng, dtype, n, 3000)
    mask = (rng.random(n) < 0.02).astype(np.uint8)
    bounds = [0, 7000, 7001, 13000, n]
    chunks = [(bounds[j], bounds[j + 1]) for j in range(4)]

    def put(a):
        if place == "device":
            return torch.from_numpy(a).cuda()
        if place == "pinned":
            return torch.from_numpy(a).pin_memory().numpy()
        return a

    states = []
    for order in (chunks, chunks[::-1], [chunks[2], chunks[0], chunks[3], chunks[1]]):
        h = device_classes(dtype)(nmaps)
        for a, b in order:
            h.update(put(keys[a:b].copy()), put(mask[a:b].copy()), a)
        look = keys_of(rng, dtype, 5000, 4000)
        look[:100] = keys[:100]
        lmask = (rng.random(len(look)) < 0.05).astype(np.uint8)
        states.append((h, look, lmask))
    o = IO.IndexHash(dtype, nmaps)
    o.update(keys, mask, 0)
    for h, look, lmask in states:
        same(state(h, put(look), put(lmask), 5), oracle_state(o, look, lmask, 5), f"{dtype} {nmaps} {place}")


def test_growth_between_calls_and_merge():
    rng = np.random.default_rng(3)
    a, b, oa, ob = device_classes("int64")(3), device_classes("int64")(3), IO.IndexHash("int64"), IO.IndexHash("int64")
    for start in range(0, 400_000, 100_000):  # 4K-slot table grows on the first call and again as distinct keys accumulate
        k = rng.integers(0, 10 ** 6, 100_000)
        a.update(k, start)
        oa.update(k, None, start)
        k2 = rng.integers(0, 10 ** 6, 50_000)
        b.update(k2, 10 ** 6 + start)
        ob.update(k2, None, 10 ** 6 + start)
    a.merge(b)
    oa.merge(ob)
    look = rng.integers(0, 10 ** 6 + 10, 30_000)
    same(state(a, look, None, -7), oracle_state(oa, look, None, -7), "growth+merge")
    assert a.extract()[0].keys().isdisjoint(a.extract()[1].keys())
    merged = {}
    for m in a.extract():
        merged.update(m)
    assert merged == oa.extract()
    assert a.offsets()[0] == 0 and len(a.offsets()) == 3


def test_merge_deviations_on_device():
    a, b = device_classes("float64")(1), device_classes("float64")(1)
    a.update(np.array([1.0, 2.0]), 0)
    b.update(np.array([np.nan, 1.0]), 2)
    a.merge(b)
    assert a.has_duplicates and a.nan_count == 1 and a.map_index(np.array([np.nan])).tolist() == [2]
    assert a.map_index_duplicates(np.array([1.0]), 0)[1].tolist() == [3]
    a, b = device_classes("int64")(1), device_classes("int64")(1)
    a.update(np.array([1, 1]), 10)
    b.update(np.array([1, 1]), 0)
    a.merge(b)
    assert a.map_index(np.array([1])).tolist() == [0] and a.map_index_duplicates(np.array([1]), 0)[1].tolist() == [1, 10, 11]
    c = device_classes("float64")(1)
    c.update(np.array([1, np.nan, 2, np.nan]), 0)
    c.update(np.array([3, np.nan, 4]), 10)
    assert c.map_index(np.array([np.nan])).tolist() == [11]


@pytest.mark.parametrize("width", G.WIDTHS)
def test_out_widths_host_and_device(width):
    import torch
    h = device_classes("int64")(1)
    h.update(np.arange(70_000, dtype=np.int64) % 40_000, -5)
    look = np.array([0, 127, 128, 300, 39_999, 50_000, -1])
    want = IO.truncate([-5, 122, 123, 295, 39_994, -1, -1], width)
    o = np.zeros(len(look), width)
    assert h.map_index(look, o) is True and np.array_equal(o, want)
    t = torch.zeros(len(look), dtype=getattr(torch, width), device="cuda")
    assert h.map_index(torch.from_numpy(look).cuda(), t) is True and np.array_equal(t.cpu().numpy(), want)
    assert h.map_index(look[:5], o[:5]) is False


def test_errors():
    h = device_classes("int64")(1)
    h.update(np.array([5.9, 7.2, 5.1]))  # forcecast by value
    assert h.has_duplicates and h.map_index(np.array([5, 7], np.int32)).tolist() == [0, 1]
    with pytest.raises(TypeError):
        h.map_index(np.array([5.0]))
    with pytest.raises(TypeError):
        h.map_index(np.array([5]), np.zeros(1, np.float32))
    other = device_classes("int64")(2)
    with pytest.raises(Exception, match="unequal maps"):
        h.merge(other)


def test_bool_keys():
    h = device_classes("bool")(1)
    h.update(np.array([True, False, True]))
    assert h.map_index(np.array([False, True])).tolist() == [1, 0] and len(h) == 3 and h.count == 2


def vector_duplicates(right_keys, left_keys, start):
    """map_index_duplicates restated with numpy (sort-based) for large inputs"""
    order = np.argsort(right_keys, kind="stable")
    sk = right_keys[order]
    lo, hi = np.searchsorted(sk, left_keys, "left"), np.searchsorted(sk, left_keys, "right")
    cnt = np.where(hi - lo > 1, hi - lo - 1, 0)
    left = np.repeat(start + np.arange(len(left_keys)), cnt)
    first = np.repeat(lo + 1, cnt)
    within = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    return left, order[first + within]


def test_duplicates_1e7_heavy():
    import torch
    rng = np.random.default_rng(11)
    rk = rng.integers(0, 2000, 10 ** 7)
    rk[: 10 ** 6] = 77  # one very heavy key
    lk = rng.integers(0, 2100, 3000)
    h = device_classes("int64")(1)
    h.update(torch.from_numpy(rk).cuda(), 0)
    left, right = h.map_index_duplicates(torch.from_numpy(lk).cuda(), 0, device=True)
    wl, wr = vector_duplicates(rk, lk, 0)
    assert left.shape[0] == len(wl) > 10 ** 7
    assert np.array_equal(left.cpu().numpy(), wl) and np.array_equal(right.cpu().numpy(), wr)


def test_1e8_right_rows():
    import torch
    g = torch.Generator(device="cuda").manual_seed(5)
    rk = torch.randint(0, 5 * 10 ** 7, (10 ** 8,), device="cuda", generator=g)
    h = device_classes("int64")(1)
    for a in range(0, 10 ** 8, 25 * 10 ** 6):
        h.update(rk[a:a + 25 * 10 ** 6], a)
    host = rk.cpu().numpy()
    uniq, first = np.unique(host, return_index=True)
    assert h.count == len(uniq) and len(h) == 10 ** 8 and h.has_duplicates
    pick = np.random.default_rng(1).integers(0, len(uniq), 10 ** 6)
    got = h.map_index(torch.from_numpy(uniq[pick]).cuda()).cpu().numpy()
    assert np.array_equal(got, first[pick])
