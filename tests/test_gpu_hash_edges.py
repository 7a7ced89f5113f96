"""The device ordered sets / counters at key edges, shard counts and table-growth boundaries, bit for bit against the oracle's
ordered set (pinned to the compiled reference on the same corpus by tests/test_set_edges_cpu.py), against the compiled reference's
own answers (tests/golden/set_edges_golden.npz) or, for sizes the oracle is too slow for, against the numpy restatement of
tests/set_cases.py.

What is covered: the key whose canonical pattern is the table's empty marker (uint64 2^64-1, -1 of a signed type) on every path
that special-cases it; every radix pass of the finalisation (row bytes 0-3, sequence bytes 0-1, shard bytes 0-1) and empty
shards; the three ways the insert table overflows and is redone (NaN / null must not be counted twice); merge with NaN / null /
sentinel; `limit`; host columns of another dtype or byte order; string sets at the hash's block boundaries and on the two
refusal paths."""
import pickle

import numpy as np
import pytest

import set_cases as S

pytestmark = pytest.mark.gpu


def to_device(a):
    """a device copy of `a`, complete before the library reads it: the library's streams do not wait for torch's"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def bits(a):
    a = np.asarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def state(s):
    keys = np.asarray(s.key_array())
    b = bits(keys).copy()
    if s.nan_count:
        assert keys[s.nan_index] != keys[s.nan_index]
        b[s.nan_index] = 0
    return dict(n=len(s), offsets=list(s.offsets()), keys=b, nan=(s.nan_count, s.nan_count and s.nan_index),
                null=(s.null_count, s.null_count and s.null_index))


def assert_same(mine, orc, what):
    a, b = state(mine), state(orc)
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: {k}: device {a[k]!r} expected {b[k]!r}"


def host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def dev_update(s, c, memspace):
    k, m = c["keys"], c["mask"]
    if memspace in ("device", "mixed"):
        k = to_device(k)
    if m is not None and memspace == "device":
        m = to_device(m)
    if m is None:
        return s.update(k, c["start_index"], return_values=c["return_values"])
    return s.update(k, m, c["start_index"], return_values=c["return_values"])


# ---- the corpus: every dtype x nmaps x memspace ------------------------------------------------------------------------------
@pytest.mark.parametrize("nmaps", S.NMAPS)
@pytest.mark.parametrize("dtype", S.DTYPES)
def test_corpus_against_oracle(dtype, nmaps, oracle):
    from vaex_b200 import superutils
    q = S.queries(dtype)
    spaces = ["host", "device", "mixed"]
    for si, (name, calls) in enumerate(S.sequences(dtype)):
        mine, orc = getattr(superutils, "ordered_set_" + dtype)(nmaps), oracle.OrderedSet(dtype, nmaps)
        for i, c in enumerate(calls):
            space = spaces[(si + i) % 3]
            a = dev_update(mine, c, space)
            b = orc.update(c["keys"], c["mask"], c["start_index"], c["return_values"])
            what = f"{name} call {i} ({space})"
            if c["return_values"]:
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), what + ": update return values"
                out = np.zeros(len(c["keys"]), np.int64)
                assert np.array_equal(mine.flatten_values(a[0], a[1], out), orc.flatten_values(b[0], b[1], np.zeros_like(out))), what
            assert_same(mine, orc, what)
        mo, oo = mine.map_ordinal(q), orc.map_ordinal(q)
        assert mo.dtype == oo.dtype and np.array_equal(mo, oo), name + ": map_ordinal"
        md = mine.map_ordinal(to_device(q))
        assert np.array_equal(host(md), oo), name + ": map_ordinal of a device column"
        assert np.array_equal(mine.isin(q), orc.isin(q)) and np.array_equal(host(mine.isin(to_device(q))), orc.isin(q)), name + ": isin"


def counts_of(keys, mask):
    """numpy: key -> count over valid non-NaN rows (canonical bit patterns as keys), nan rows, null rows"""
    keys = np.asarray(keys)
    valid = np.ones(len(keys), bool) if mask is None else ~mask
    isnan = np.isnan(keys) if keys.dtype.kind == "f" else np.zeros(len(keys), bool)
    u, n = np.unique(bits(keys[valid & ~isnan]), return_counts=True)
    return dict(zip(u.tolist(), n.tolist())), int((valid & isnan).sum()), int((~valid).sum())


def counter_state(c):
    keys = np.asarray(c.key_array())
    counts = c.counts()
    skip = int(c.nan_count > 0) + int(c.null_count > 0)
    got = dict(zip(bits(keys[skip:]).tolist(), counts[skip:].tolist()))
    nan = int(counts[0]) if c.nan_count else 0
    null = int(counts[c.null_index]) if c.null_count else 0
    return got, nan, null


@pytest.mark.parametrize("nmaps", [1, 257])
@pytest.mark.parametrize("dtype", S.DTYPES)
def test_counter_corpus(dtype, nmaps):
    from vaex_b200 import superutils
    for name, calls in S.sequences(dtype):
        c = getattr(superutils, "counter_" + dtype)(nmaps)
        allk, allm = [], []
        for call in calls:
            dev_update(c, dict(call, return_values=False), "device" if name == "run" else "host")
            allk.append(call["keys"])
            allm.append(np.zeros(len(call["keys"]), bool) if call["mask"] is None else call["mask"])
        want, nan, null = counts_of(np.concatenate(allk), np.concatenate(allm))
        got, gnan, gnull = counter_state(c)
        assert (c.nan_count, c.null_count) == (nan, null) == (gnan, gnull), name
        assert got == want, name


def test_golden_vectors_of_the_compiled_reference():
    """tests/golden/set_edges_golden.npz: the compiled reference run over the corpus (without -0.0), nmaps 1 / 3 / 257"""
    import golden_util
    from vaex_b200 import superutils
    gold = golden_util.load_set_edges()
    assert len(gold) > 50
    for name, g in sorted(gold.items()):
        dtype, nmaps = str(g["dtype"]), int(g["nmaps"])
        if name.startswith("merge_"):
            continue
        s = getattr(superutils, "ordered_set_" + dtype)(nmaps)
        for i in range(int(g["ncalls"])):
            k = g[f"c{i}_keys"]
            m = g[f"c{i}_mask"] if f"c{i}_mask" in g else None
            si, rv = (int(x) for x in g[f"c{i}_opts"])
            r = s.update(k, m, si, return_values=bool(rv)) if m is not None else s.update(k, si, return_values=bool(rv))
            if rv:
                assert np.array_equal(r[0], g[f"c{i}_values"]) and np.array_equal(r[1], g[f"c{i}_map"]), f"{name} call {i}"
        st = state(s)
        assert st["offsets"] == g["offsets"].tolist(), name
        assert np.array_equal(st["keys"], g["keys"]), name
        assert st["nan"] == tuple(g["nan"].tolist()) and st["null"] == tuple(g["null"].tolist()), name
        mo = s.map_ordinal(g["query"])
        assert mo.dtype == g["query_ordinals"].dtype and np.array_equal(mo, g["query_ordinals"]), name
        assert np.array_equal(s.isin(g["query"]), g["query_isin"]), name


# ---- radix passes of the finalisation ----------------------------------------------------------------------------------------
def test_three_hundred_update_calls(oracle):
    """more than 256 calls on one set: the second byte of the call sequence is sorted on; NaN and null first seen late"""
    from vaex_b200 import superutils
    rng = np.random.default_rng(300)
    mine, orc = superutils.ordered_set_float64(3), oracle.OrderedSet("float64", 3)
    for call in range(300):
        k = rng.integers(0, 5000, 40).astype("f8")
        k[:2] = 6000 - call  # new keys in every call, at rows 0 and 1, so that only the call number orders them
        m = None
        if call == 270:
            k[5] = np.nan
        if call >= 280:
            m = np.zeros(len(k), bool)
            m[7] = True
        mine.update(k, m, -1) if m is not None else mine.update(k, -1)
        orc.update(k, m, -1, False)
    assert_same(mine, orc, "300 calls")
    q = np.concatenate([np.arange(6001, dtype="f8"), [np.nan]])
    assert np.array_equal(mine.map_ordinal(q), orc.map_ordinal(q))


def test_call_of_2_24_plus_2_16_rows_with_late_first_occurrences():
    """one call whose new keys first appear in the last 2^16 rows: row bytes 2 and 3 decide their order; the null arrives in a
    later call (its tag is remapped behind the largest row)"""
    from vaex_b200 import superutils
    import torch
    n0, n1 = 1 << 24, 1 << 16
    rng = np.random.default_rng(24)
    pool = np.arange(1000, dtype=np.int64) * 7919 - 3_000_000
    head = pool[rng.integers(0, 1000, n0)]
    head[:1000] = pool  # every pool key is seen in the first 1000 rows
    tail = rng.permutation(n1).astype(np.int64) * 13 + 10 ** 9
    tail[::97] = -1  # the sentinel first appears late as well
    big = np.concatenate([head, tail])
    later = np.array([5, -1, 2 ** 40, 7, 5], np.int64)
    later_mask = np.array([0, 0, 0, 1, 0], bool)
    s = superutils.ordered_set_int64(7)
    s.update(to_device(big), -1)
    s.update(later, later_mask, -1)
    keys, offsets, null_pos, null_count = S.restate([(big, None), (later, later_mask)], "int64", 7)
    assert s.offsets() == offsets
    assert np.array_equal(s.key_array(), keys)
    assert (s.null_count, s.null_index) == (null_count, null_pos)
    probe = np.concatenate([tail[:5000], pool[:100], later])
    pos = {k: i for i, k in enumerate(keys.tolist()) if i != null_pos}  # ordinal == position in key_array
    assert s.map_ordinal(probe).tolist() == [pos.get(k, -1) for k in probe.tolist()]


@pytest.mark.parametrize("nmaps", [257, 32767])
def test_many_shards_few_keys(nmaps, oracle):
    """nmaps > 256 sorts on the second shard byte; with a handful of keys almost every shard is empty"""
    from vaex_b200 import superutils
    for dtype in ("int64", "int16", "float32"):
        k = np.concatenate([S.edge_values(dtype)[:9], S.nan_values(dtype)[:1]])
        m = np.zeros(len(k), bool)
        m[2] = True
        mine, orc = getattr(superutils, "ordered_set_" + dtype)(nmaps), oracle.OrderedSet(dtype, nmaps)
        mine.update(k, m, 0)
        orc.update(k, m, 0, False)
        assert_same(mine, orc, dtype)
        assert np.array_equal(mine.map_ordinal(k), orc.map_ordinal(k))


# ---- overflow and redo --------------------------------------------------------------------------------------------------------
def _check_overflow_case(kind, chunks):
    """chunks: list of (device float64 keys, device bool mask) update calls; checks against torch-side counts / first occurrences"""
    import torch
    from vaex_b200 import superutils
    s = getattr(superutils, ("counter_" if kind == "counter" else "ordered_set_") + "float64")(1)
    torch.cuda.synchronize()  # the columns were generated on torch's stream
    nan = null = 0
    order = []
    for k, m in chunks:
        s.update(k, m, -1)
        valid = ~m
        isnan = torch.isnan(k)
        nan += int((valid & isnan).sum())
        null += int(m.sum())
        order.append(k[valid & ~isnan])
    assert (s.nan_count, s.null_count) == (nan, null), "NaN / null counted once per row, also across a redo"
    allk = torch.cat(order)
    u, inv, cnt = torch.unique(allk, return_inverse=True, return_counts=True)
    if kind == "counter":
        keys, counts = s.key_array(), s.counts()
        assert counts[0] == nan and counts[1] == null
        got_k, got_c = torch.from_numpy(keys[2:]).cuda(), torch.from_numpy(counts[2:]).cuda()
        o = torch.argsort(got_k)
        assert torch.equal(got_k[o], u) and torch.equal(got_c[o], cnt), "counts equal np.unique(return_counts=True)"
    else:
        # first-occurrence order of the distinct keys; NaN and null (both seen in the first call) right behind the first call's
        # keys (start_index -1: NaN before null; nmaps 1: shard 0 is everything)
        pos = torch.arange(len(allk), device=allk.device)
        first = torch.full((len(u),), len(allk), dtype=torch.int64, device=allk.device).scatter_reduce(0, inv, pos, reduce="amin")
        want = u[torch.argsort(first)]
        n0 = int((first < len(order[0])).sum())
        keys = torch.from_numpy(s.key_array()).cuda()
        assert len(keys) == len(u) + 2
        assert (s.nan_index, s.null_index) == (n0, n0 + 1)
        assert torch.equal(torch.cat([keys[:n0], keys[n0 + 2:]]), want)


def _with_specials(k, gen, nan_frac=0.01, mask_frac=0.01):
    import torch
    k = k.clone()
    r = torch.rand(len(k), generator=gen, device=k.device)
    k[r < nan_frac] = float("nan")
    m = (r > 1 - mask_frac)
    k[:4] = torch.arange(4, device=k.device, dtype=k.dtype) + 0.5  # some keys seen before any special
    m[:4] = False
    return k, m


@pytest.mark.parametrize("kind", ["set", "counter"])
def test_overflow_dirty_second_call(kind):
    """the second call on a dirty set sizes its table for its own rows only (known = 0): as many new keys as the first call
    overflow it, the range is redone after a growth"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(1)
    n = 1_000_000
    a = _with_specials(torch.randperm(n, generator=g, device="cuda").double() * 3, g)
    b = _with_specials(torch.randperm(n, generator=g, device="cuda").double() * 3 + 1, g)
    _check_overflow_case(kind, [a, b])


@pytest.mark.parametrize("kind", ["set", "counter"])
def test_overflow_one_call_beyond_the_sizing_cap(kind):
    """one call of 3 * 2^21 distinct keys: the up-front sizing is capped at 2^22 slots"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(2)
    n = 3 << 21
    k = torch.randperm(n, generator=g, device="cuda").double() * 0.5 - 1e6
    _check_overflow_case(kind, [_with_specials(k, g)])


@pytest.mark.parametrize("kind", ["set", "counter"])
def test_overflow_in_the_second_sub_range(kind):
    """a call of more than 2^26 rows is inserted in 2^26-row ranges: few distinct keys in the first, 2^22 new ones in the second,
    which overflows; only that range is redone"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(3)
    n0, n1 = 1 << 26, 1 << 22
    k = torch.cat([(torch.arange(n0, device="cuda") % 1000).double(), torch.randperm(n1, generator=g, device="cuda").double() + 5000.5])
    _check_overflow_case(kind, [_with_specials(k, g, nan_frac=1e-4, mask_frac=1e-4)])


# ---- the key whose pattern is the empty marker --------------------------------------------------------------------------------
SENTINEL_TYPES = ["uint64", "int64", "int32", "int16", "int8"]


@pytest.mark.parametrize("dtype", SENTINEL_TYPES)
def test_sentinel_merge_from_keys_pickle_counter(dtype, oracle):
    from vaex_b200 import superutils
    sent = S.sentinel(dtype)
    cls = getattr(superutils, "ordered_set_" + dtype)
    other = np.array([3, sent, 4, sent], dtype)
    # merge: the sentinel only in the other set
    a, b = cls(3), cls(3)
    a.update(np.array([1, 2, 3], dtype))
    b.update(other)
    a.merge([b])
    assert len(a) == 5 and a.map_ordinal(np.array([sent], dtype))[0] >= 0
    assert a.key_array()[a.map_ordinal(np.array([sent], dtype))[0]] == sent
    assert a.isin(np.array([sent, 9], dtype)).tolist() == [True, False]
    # from_keys and pickle: the sentinel first, last, next to the null slot
    for keys, null_index in (([sent, 1, 2], -1), ([1, 2, sent], -1), ([sent, 5, 6], 1), ([7, sent, 8], 2)):
        k = np.array(keys, dtype)
        null_count = int(null_index >= 0)
        s = cls(k, null_index, 0, null_count, "fp")
        o = oracle.OrderedSet.from_keys(k, null_index, 0, null_count)
        assert_same(s, o, f"from_keys {keys} null_index={null_index}")
        q = np.array([sent, 1, 2, 5, 6, 7, 8, 9], dtype)
        assert np.array_equal(s.map_ordinal(q), o.map_ordinal(q))
        clone = pickle.loads(pickle.dumps(s))
        assert_same(clone, o, "pickle round trip")
        assert np.array_equal(clone.map_ordinal(q), o.map_ordinal(q))
    # counter: the sentinel's occurrences, also through a merge
    c1, c2 = getattr(superutils, "counter_" + dtype)(3), getattr(superutils, "counter_" + dtype)(3)
    c1.update(np.array([sent, 1, sent, sent], dtype), np.array([0, 0, 0, 1], bool))
    c2.update(other)
    c1.merge([c2])
    got, _, null = counter_state(c1)
    assert got == {int(bits(np.array([sent], dtype))[0]): 4, 1: 1, 3: 1, 4: 1} and null == 1


def test_sentinel_in_groupby_fused_and_combined():
    """Frame.groupby: the fused probe (B200_BINNER_HASH) and the two-key combined code (k_set_combine) with the sentinel, NaN and
    masked keys; value_counts / unique"""
    from vaex_b200 import agg
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(31)
    n = 20_000
    k1 = rng.choice(np.array([-1, 0, 1, 2 ** 62, -(2 ** 63)], np.int64), n)
    k1m = np.ma.array(k1, mask=rng.random(n) < 0.05)
    k2 = rng.choice(np.array([np.nan, 0.5, -0.0, np.inf, 1e300]), n)
    u64 = rng.choice(np.array([2 ** 64 - 1, 0, 2 ** 63], np.uint64), n)
    df = Frame(dict(k1=k1m, k2=k2, u=u64, v=np.ones(n)))
    for col, data in (("k1", k1m), ("u", u64)):
        out = df.groupby(col, agg={"v": "count"})
        got = {(None if np.ma.is_masked(k) else int(k)): int(c) for k, c in zip(out[col], out["v_count"])}
        valid = np.ma.getmaskarray(data) if np.ma.isMaskedArray(data) else np.zeros(n, bool)
        raw = np.asarray(np.ma.getdata(data))
        u, c = np.unique(raw[~valid], return_counts=True)
        want = dict(zip(u.tolist(), c.tolist()))
        if valid.any():
            want[None] = int(valid.sum())
        assert got == want, col
        keys, counts = df.value_counts(col)
        assert {(None if k is None else int(k)): int(c) for k, c in zip(keys, counts)} == want, col
    out = df.groupby(["k1", "k2"], agg=[agg.count()], combine=True)
    got = {}
    for a, b, c in zip(out["k1"], out["k2"], out["count"]):
        got[(None if np.ma.is_masked(a) else int(a), "nan" if b != b else float(b).hex())] = int(c)
    want = {}
    for a, am, b in zip(k1.tolist(), np.ma.getmaskarray(k1m).tolist(), k2.tolist()):
        key = (None if am else a, "nan" if b != b else float(b).hex())
        want[key] = want.get(key, 0) + 1
    assert got == want
    assert sorted(int(x) for x in df.unique("u")) == sorted({int(x) for x in u64.tolist()})


# ---- merge with specials -------------------------------------------------------------------------------------------------------
def test_merge_with_specials_keeps_ordinals_distinct():
    """Deviation from the reference (DESIGN.md section 3): a key merged in after a NaN / null takes the next free ordinal, and a
    NaN / null first seen through a merge gets its own ordinal, behind the keys of the merge.  The reference hands out the NaN's
    ordinal twice in the first case and leaves nan_index at 0x7fffffff in the second (tests/test_set_edges_cpu.py)."""
    from vaex_b200 import superutils
    a, b = superutils.ordered_set_float64(1), superutils.ordered_set_float64(1)
    a.update(np.array([1.0, np.nan]))
    b.update(np.array([5.0]))
    a.merge([b])
    assert a.map_ordinal(np.array([1.0, np.nan, 5.0])).tolist() == [0, 1, 2]
    import golden_util
    gold = golden_util.load_set_edges()
    g = gold["merge_nan_left"]
    assert g["query_ordinals"].tolist() == [0, 1, 1], "the reference hands the NaN's ordinal to 5.0 as well"
    assert a.map_ordinal(g["query"]).tolist() == [0, 2, 1]
    g = gold["merge_nan_right"]
    assert g["nan"].tolist() == [1, 0x7FFFFFFF], "the reference never sets nan_index for a NaN first seen through a merge"
    a, b = superutils.ordered_set_float64(1), superutils.ordered_set_float64(1)
    a.update(np.array([1.0]))
    b.update(np.array([7.0, np.nan, 2.0]), np.array([0, 0, 1], bool))
    a.merge([b])
    assert (a.nan_count, a.nan_index, a.null_count, a.null_index) == (1, 2, 1, 3)
    assert a.map_ordinal(np.array([1.0, 7.0, np.nan])).tolist() == [0, 1, 2]
    # specials on both sides: counts add, ordinals stay where they were
    a, b = superutils.ordered_set_float64(3), superutils.ordered_set_float64(3)
    a.update(np.array([np.nan, 4.0, 9.0]), np.array([0, 0, 1], bool))
    b.update(np.array([np.nan, 4.0, 8.0, 8.0]), np.array([0, 0, 1, 0], bool))
    nan_i, null_i = a.nan_index, a.null_index
    a.merge([b])
    assert (a.nan_count, a.null_count, a.nan_index, a.null_index) == (2, 2, nan_i, null_i) and len(a) == 4
    ords = a.map_ordinal(np.array([4.0, 8.0, np.nan]))
    assert len(set(ords.tolist()) | {null_i}) == 4


@pytest.mark.parametrize("dtype", ["float64", "int64"])
def test_counter_merge_with_specials(dtype):
    from vaex_b200 import superutils
    sent = S.sentinel(dtype)
    spec = np.nan if dtype == "float64" else sent
    c1, c2 = getattr(superutils, "counter_" + dtype)(3), getattr(superutils, "counter_" + dtype)(3)
    k1 = np.array([1, spec, 2, spec, 3], dtype)
    m1 = np.array([0, 0, 0, 0, 1], bool)
    k2 = np.array([spec, 2, 5, 5, 6], dtype)
    m2 = np.array([0, 0, 0, 0, 1], bool)
    c1.update(k1, m1)
    c2.update(k2, m2)
    c1.merge([c2])
    want, nan, null = counts_of(np.concatenate([k1, k2]), np.concatenate([m1, m2]))
    got, gnan, gnull = counter_state(c1)
    assert got == want and (gnan, gnull) == (nan, null) == (c1.nan_count, c1.null_count)


# ---- limit ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["int64", "uint64", "float64", "int8"])
def test_limit_against_oracle(dtype, oracle):
    from vaex_b200 import superutils
    calls = [c for _, seq in S.sequences(dtype) for c in seq]
    for limit in (0, 3, 40):
        mine, orc = getattr(superutils, "ordered_set_" + dtype)(3, limit), oracle.OrderedSet(dtype, 3, limit)
        for i, c in enumerate(calls):
            c = dict(c, return_values=False)
            dev_update(mine, c, "device" if i % 2 else "host")
            orc.update(c["keys"], c["mask"], c["start_index"], False)
            assert_same(mine, orc, f"limit={limit} call {i}")
        with pytest.raises(RuntimeError, match="limit"):
            mine.update(calls[0]["keys"], 0, return_values=True)


# ---- host marshalling: dtype and byte order -------------------------------------------------------------------------------------
def test_host_columns_are_converted_by_value():
    """like the reference's py::array_t<T> forcecast (answers pinned in tests/test_set_edges_cpu.py): big-endian columns insert
    their numbers, columns of another dtype are converted by value; a device column of another kind is refused"""
    import torch
    from vaex_b200 import superutils
    s = superutils.ordered_set_int64(1)
    s.update(np.array([1, 2, 3], ">i8"))
    assert s.key_array().tolist() == [1, 2, 3]
    s = superutils.ordered_set_int64(1)
    s.update(np.array([1.7, 2.2]))
    assert s.key_array().tolist() == [1, 2]
    assert s.map_ordinal(np.array([2, 1], ">i8")).tolist() == [1, 0]
    assert s.isin(np.array([2.9, 5.0])).tolist() == [True, False]
    s = superutils.ordered_set_float32(1)
    s.update(np.array([1.5, -2.25], ">f4"))
    assert s.key_array().tolist() == [1.5, -2.25]
    rng = np.random.default_rng(8)
    for dtype in ("float64", "float32", "int64", "int32", "int16", "uint64", "uint32", "uint16"):
        k = S.columns(dtype)[0][1]
        native, swapped = getattr(superutils, "ordered_set_" + dtype)(7), getattr(superutils, "ordered_set_" + dtype)(7)
        native.update(k, -1)
        swapped.update(k.astype(k.dtype.newbyteorder()), -1)
        assert_same(swapped, native, dtype + " big-endian")
        q = np.concatenate([k[:100], rng.permutation(k)[:100]])
        assert np.array_equal(native.map_ordinal(q.astype(q.dtype.newbyteorder())), native.map_ordinal(q))
        assert np.array_equal(native.isin(q.astype(q.dtype.newbyteorder())), native.isin(q))
        c = getattr(superutils, "counter_" + dtype)(1)
        c.update(k.astype(k.dtype.newbyteorder()))
        assert counter_state(c) == counts_of(k, None)
    s = superutils.ordered_set_int64(1)
    with pytest.raises(TypeError):
        s.update(torch.zeros(4, dtype=torch.float64, device="cuda"))
    with pytest.raises(TypeError):
        s.map_ordinal(torch.zeros(4, dtype=torch.float64, device="cuda"))
    s.update(torch.tensor([5, 6], dtype=torch.int64, device="cuda"))
    assert s.key_array().tolist() == [5, 6]


def test_big_endian_columns_in_groupby_and_value_counts():
    """a big-endian key column gives the same groups, group order and counts as the native one (pass 1 builds the set from the
    converted keys, pass 2's fused probe reads the column with its byte swap)"""
    from vaex_b200.frame import Frame
    rng = np.random.default_rng(9)
    n = 30_000
    for dt in ("i8", "f8", "i4", "u2"):
        k = rng.integers(-50, 50, n).astype(dt)
        if dt == "f8":
            k[::101] = np.nan
        v = rng.normal(size=n)
        a = Frame(dict(k=k, v=v)).groupby("k", agg={"v": ["sum", "count"]})
        b = Frame(dict(k=k.astype(k.dtype.newbyteorder()), v=v)).groupby("k", agg={"v": ["sum", "count"]})
        assert np.array_equal(np.asarray(a["k"], "f8"), np.asarray(b["k"], "f8"), equal_nan=True), dt
        assert np.array_equal(a["v_count"], b["v_count"]) and np.allclose(a["v_sum"], b["v_sum"]), dt
        ka, ca = Frame(dict(k=k)).value_counts("k")
        kb, cb = Frame(dict(k=k.astype(k.dtype.newbyteorder()))).value_counts("k")
        assert np.array_equal(ca, cb) and str(ka) == str(kb), dt


# ---- strings ----------------------------------------------------------------------------------------------------------------------
def _words():
    out = ["", "\0", "a\0b", "\0\0\0\0\0\0\0\0", "x" * 1000, "äß€" * 7]
    for n in range(18):
        out.append("".join(chr(97 + (i * 7 + n) % 26) for i in range(n)))
        out.append("\0" * (n // 2) + "q" * (n - n // 2))
    return out


@pytest.mark.parametrize("nmaps", [1, 3, 257])
def test_string_edges_against_oracle(nmaps, oracle):
    """empty and NUL-carrying strings, every length 0-17 around the 8-byte block / tail split, long strings; sliced arrow arrays
    (offsets not starting at 0), string and large_string offsets; nulls across table and pool growth"""
    import pyarrow as pa
    from vaex_b200 import superutils
    rng = np.random.default_rng(nmaps)
    words = _words()
    s, o = superutils.ordered_set_string(nmaps), oracle.StringOrderedSet(nmaps)
    for call in range(5):
        n = [50, 3000, 1, 20_000, 400][call]
        vals = [words[i] if i < len(words) else f"w{i}-{call}" for i in rng.integers(0, len(words) + 40 + 3000 * (call == 3), n)]
        if call >= 2:
            vals = [None if rng.random() < 0.05 else v for v in vals]
        arr = pa.array(["pad"] * 3 + vals, type=pa.large_string() if call % 2 else pa.string()).slice(3)
        a = s.update(arr, 0, return_values=True)
        b = o.update(vals, 0, True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), f"call {call}"
        assert s.keys() == o.keys() and s.offsets() == o.offsets() and len(s) == len(o)
        assert s.null_index == o.null_index
    probe = words + [None, "not a member", "w9999-9"]
    assert s.map_ordinal(probe).tolist() == o.map_ordinal(probe).tolist()


def test_string_refusals_leave_the_set_usable(oracle):
    """a string whose 64-bit hash is the table's empty marker, and a string that shares its hash with a member, are refused with
    the library's messages; the set keeps every other key and later calls work"""
    from vaex_b200 import superutils
    empty = S.ascii_string_with_hash(2 ** 64 - 1)
    member = "abcdefgh12345678"
    twin = S.ascii_collision(member)
    s, o = superutils.ordered_set_string(3), oracle.StringOrderedSet(3)
    s.update(["x", member, "yy"])
    o.update(["x", member, "yy"])
    with pytest.raises(RuntimeError, match="reserved empty pattern"):
        s.update([empty])
    with pytest.raises(RuntimeError, match="share one 64-bit hash"):
        s.update([twin])
    s.update(["z", None, "x"])
    o.update(["z", None, "x"])
    assert s.keys() == o.keys() and s.offsets() == o.offsets()
    probe = ["x", member, "yy", "z", None, twin, empty, "nope"]
    want = o.map_ordinal(probe[:5] + ["nope", "nope", "nope"]).tolist()
    assert s.map_ordinal(probe).tolist() == want
