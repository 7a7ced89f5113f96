"""The oracle's ordered set (oracle/binstats_oracle.c, oracle.OrderedSet) against the compiled reference's ordered_set_<T> on the
edge corpus of tests/set_cases.py, bit for bit wherever the reference's answer does not depend on its container; plus the numpy
restatement the big GPU cases use, checked against the oracle, and the std::hash inverse the string-refusal tests use.

Deviations of the reference that depend on its container are asserted as such, with the reference's actual output in the
message: +0.0 / -0.0 (merged in small tables, kept apart in larger ones) and the order in which `merge` appends keys."""
import numpy as np
import pytest

import set_cases as S


def bits(a):
    a = np.asarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def ref_update(s, c):
    kw = dict(start_index=c["start_index"], return_values=c["return_values"])
    if c["mask"] is None:
        return s.update(c["keys"], **kw)
    return s.update(c["keys"], np.ascontiguousarray(c["mask"], bool), **kw)


def orc_update(s, c):
    return s.update(c["keys"], c["mask"], c["start_index"], c["return_values"])


def state(s):
    keys = np.asarray(s.key_array())
    b = bits(keys).copy()
    if s.nan_count:
        assert keys[s.nan_index] != keys[s.nan_index]
        b[s.nan_index] = 0
    return dict(n=len(s), offsets=list(s.offsets()), keys=b, nan=(s.nan_count, s.nan_count and s.nan_index), null=(s.null_count, s.null_count and s.null_index))


def assert_same(mine, ref, what):
    a, b = state(mine), state(ref)
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs: oracle {a[k]!r} reference {b[k]!r}"


@pytest.mark.parametrize("nmaps", S.NMAPS)
@pytest.mark.parametrize("dtype", S.DTYPES)
def test_oracle_matches_reference_on_edge_corpus(dtype, nmaps, oracle, ref):
    q = S.queries(dtype, zeros=False)
    for name, calls in S.sequences(dtype, zeros=False):
        o, r = oracle.OrderedSet(dtype, nmaps), ref.ordered_set(dtype, nmaps)
        for i, c in enumerate(calls):
            a, b = orc_update(o, c), ref_update(r, c)
            if c["return_values"]:
                assert np.array_equal(a[0], np.asarray(b[0])) and np.array_equal(a[1], np.asarray(b[1])), f"{name} call {i}: update return values"
            assert_same(o, r, f"{dtype} nmaps={nmaps} {name} call {i}")
        mo, mr = o.map_ordinal(q), np.asarray(r.map_ordinal(q))
        assert mo.dtype == mr.dtype and np.array_equal(mo, mr), f"{name}: map_ordinal"
        assert np.array_equal(o.isin(q), np.asarray(r.isin(q))), f"{name}: isin"


@pytest.mark.parametrize("dtype", S.DTYPES)
def test_from_keys_matches_reference(dtype, oracle, ref):
    """ordered_set_<T>(keys, null_index, nan_count, null_count, fingerprint) with the sentinel, NaN payloads and the null slot
    first / last / absent"""
    keys = np.unique(S.edge_values(dtype, zeros=False))
    nans = S.nan_values(dtype)
    variants = [(keys, -1, 0, 0)]
    if len(keys) > 2:
        variants += [(keys, 0, 0, 1), (keys, len(keys) - 1, 0, 1)]
    if len(nans):
        kn = np.concatenate([keys, nans[2:3]])
        variants += [(kn, -1, 1, 0), (kn, 0, 1, 1)]
    q = S.queries(dtype, zeros=False)
    for k, null_index, nan_count, null_count in variants:
        o = oracle.OrderedSet.from_keys(k, null_index, nan_count, null_count)
        r = ref.ordered_set_from_keys(k, null_index, nan_count, null_count)
        assert_same(o, r, f"from_keys null_index={null_index} nan={nan_count}")
        assert np.array_equal(o.map_ordinal(q), np.asarray(r.map_ordinal(q)))


@pytest.mark.parametrize("dtype", ["int64", "uint64", "float64", "int8"])
def test_limit_matches_reference(dtype, oracle, ref):
    """limit: once count() >= limit before a call, the whole flush of that call is skipped (NaN / null still counted); mixing
    limit with return_values raises"""
    calls = [c for _, seq in S.sequences(dtype, zeros=False) for c in seq]
    for limit in (0, 3, 40):
        o, r = oracle.OrderedSet(dtype, 3, limit), ref.ordered_set(dtype, 3, limit)
        for c in calls:
            c = dict(c, return_values=False)
            orc_update(o, c)
            ref_update(r, c)
            assert_same(o, r, f"limit={limit}")
        with pytest.raises(RuntimeError):
            o.update(calls[0]["keys"], None, 0, True)
        with pytest.raises(RuntimeError):
            r.update(calls[0]["keys"], return_values=True)


@pytest.mark.parametrize("n_extra, nan, null", [(125, 1, 1), (126, 1, 1), (127, 0, 0), (32765, 1, 1), (32766, 1, 0), (32767, 0, 0), (32766, 1, 1)])
def test_map_ordinal_dtype_boundaries(n_extra, nan, null, oracle, ref):
    """the ordinal dtype steps at 2^7 / 2^15 entries; the NaN and null slots count"""
    k = np.arange(n_extra, dtype=np.float64) * 3 + 1
    m = None
    if nan:
        k = np.concatenate([k, [np.nan]])
    if null:
        k = np.concatenate([k, [7.0]])
        m = np.zeros(len(k), bool)
        m[-1] = True
    o, r = oracle.OrderedSet("float64", 2), ref.ordered_set("float64", 2)
    c = dict(keys=k, mask=m, start_index=0, return_values=False)
    orc_update(o, c)
    ref_update(r, c)
    assert len(o) == n_extra + nan + null
    a, b = o.map_ordinal(k), np.asarray(r.map_ordinal(k))
    assert a.dtype == b.dtype and np.array_equal(a, b)


def test_zero_signs_depend_on_the_reference_table_size(oracle, ref):
    """Deviation: the oracle (and the device) keep +0.0 and -0.0 apart, as distinct bit patterns.  The reference compares keys
    with == but hashes their bits, so whether the two zeros meet depends on where its container puts them."""
    for dtype in ("float64", "float32"):
        z = np.array([0.0, -0.0], dtype)
        for nmaps in (1, 3, 7):
            o, r = oracle.OrderedSet(dtype, nmaps), ref.ordered_set(dtype, nmaps)
            o.update(z, None, 0, False)
            r.update(z)
            assert len(o) == 2, "the oracle keeps +0.0 and -0.0 apart"
            assert len(r) in (1, 2), f"reference: {len(r)} keys for [0.0, -0.0] ({dtype}, nmaps={nmaps})"
        big = np.concatenate([np.arange(1, 1001, dtype=dtype), z])
        o, r = oracle.OrderedSet(dtype, 1), ref.ordered_set(dtype, 1)
        o.update(big, None, 0, False)
        r.update(big)
        assert len(o) == 1002, f"reference after 1000 other keys: {len(r)} keys"


def test_merge_with_specials_reference_semantics(oracle, ref):
    """The reference's merge emplaces a new key with ordinal maps[i].size() and ignores the NaN / null ordinal offset of shard 0,
    and never sets nan_value for a NaN first seen through a merge; the oracle restates both.  The device keeps ordinals distinct
    instead (DESIGN.md section 3, tests/test_gpu_hash_edges.py)."""
    for lib in (oracle, ref):
        mk = (lambda: oracle.OrderedSet("float64", 1)) if lib is oracle else (lambda: ref.ordered_set("float64", 1))
        a, b = mk(), mk()
        a.update(np.array([1.0, np.nan]), *(() if lib is ref else (None, 0, False)))
        b.update(np.array([5.0]), *(() if lib is ref else (None, 0, False)))
        a.merge([b])
        assert np.asarray(a.map_ordinal(np.array([5.0, np.nan]))).tolist() == [1, 1], lib
        a, b = mk(), mk()
        a.update(np.array([1.0]), *(() if lib is ref else (None, 0, False)))
        b.update(np.array([7.0, np.nan]), *(() if lib is ref else (None, 0, False)))
        a.merge([b])
        assert (a.nan_count, a.nan_index) == (1, 0x7FFFFFFF), lib


def test_merge_order_is_container_order_in_the_reference(oracle, ref):
    """merge appends the other set's new keys; the oracle in the other set's insertion order, the reference in its container's
    iteration order.  The union of keys, the counts and the keys already present agree."""
    ka = np.arange(0, 60, dtype=np.int64) * 11
    kb = np.concatenate([[-1], np.arange(30, 120, dtype=np.int64) * 11])
    o, ob = oracle.OrderedSet("int64", 3), oracle.OrderedSet("int64", 3)
    r, rb = ref.ordered_set("int64", 3), ref.ordered_set("int64", 3)
    o.update(ka, None, 0, False), ob.update(kb, None, 0, False)
    r.update(ka), rb.update(kb)
    o.merge([ob])
    r.merge([rb])
    assert len(o) == len(r) == len(np.union1d(ka, kb))
    assert sorted(o.key_array().tolist()) == sorted(np.asarray(r.key_array()).tolist())
    assert np.array_equal(o.map_ordinal(ka), np.asarray(r.map_ordinal(ka))), "keys present before the merge keep their ordinals"
    assert o.offsets() == list(r.offsets())


def test_host_keys_are_converted_by_value_in_the_reference(ref):
    """pybind11's forcecast of py::array_t<T>: big-endian columns and columns of another dtype are converted by value.  The device
    set's host marshalling does the same (tests/test_gpu_hash_edges.py checks it against these answers)."""
    r = ref.ordered_set("int64", 1)
    r.update(np.array([1, 2, 3], ">i8"))
    assert np.asarray(r.key_array()).tolist() == [1, 2, 3]
    r = ref.ordered_set("int64", 1)
    r.update(np.array([1.7, 2.2]))
    assert np.asarray(r.key_array()).tolist() == [1, 2]
    assert np.asarray(r.map_ordinal(np.array([2, 1], ">i8"))).tolist() == [1, 0]
    assert np.asarray(r.isin(np.array([2.9, 5.0]))).tolist() == [True, False]
    r = ref.ordered_set("float32", 1)
    r.update(np.array([1.5, -2.25], ">f4"))
    assert np.asarray(r.key_array()).tolist() == [1.5, -2.25]


@pytest.mark.parametrize("nmaps", [1, 3, 257, 1000])
def test_numpy_restatement_matches_oracle(nmaps, oracle):
    """the restatement used for the big GPU cases: per shard the rank of first occurrence; a null joins shard 0 at the end of the
    call that first saw it"""
    rng = np.random.default_rng(nmaps)
    for dtype in ("int64", "int16", "uint64"):
        calls = []
        o = oracle.OrderedSet(dtype, nmaps)
        for ci in range(4):
            n = int(rng.integers(1, 5000))
            k = rng.integers(-3000, 3000, n).astype(dtype)
            if ci == 3:
                k[-50:] = np.arange(50) * 7919 + 10 ** 4  # first occurrences late in the call
            m = (rng.random(n) < 0.03) if ci >= 1 else None
            calls.append((k, m))
            o.update(k, m, -1, False)
            keys, offsets, null_pos, null_count = S.restate(calls, dtype, nmaps)
            assert offsets == o.offsets() and np.array_equal(keys, o.key_array()), (dtype, ci)
            assert null_count == o.null_count and (null_pos is None or null_pos == o.null_index)


def test_string_hash_inverse(oracle):
    """set_cases.last_block_for undoes std::hash<string_view> (64-bit Murmur-2) on one 8-byte block"""
    rng = np.random.default_rng(5)
    for _ in range(50):
        prefix = bytes(rng.integers(0, 256, 8 * int(rng.integers(0, 3)), dtype=np.uint8))
        target = int(rng.integers(0, 2 ** 63)) * 2 + 1
        assert oracle.string_hash(prefix + S.last_block_for(prefix, target)) == target
    s = S.ascii_string_with_hash(2 ** 64 - 1)
    assert len(s) == 16 and oracle.string_hash(s.encode()) == 2 ** 64 - 1
    a = "abcdefgh12345678"
    b = S.ascii_collision(a)
    assert a != b and oracle.string_hash(a.encode()) == oracle.string_hash(b.encode())

