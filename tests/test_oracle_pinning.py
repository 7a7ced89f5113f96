"""Pin the oracle (oracle/binstats_oracle.c) — CPU only.

 1. against the golden vectors generated from the compiled, unmodified reference (tests/golden/, always available);
 2. against the compiled reference itself (oracle/_ref) on fresh random cases when it is present in this container.
The oracle is the checker of every GPU parity test, so it has to be right first."""
import numpy as np
import pytest

import golden_util
from helpers import random_case, same, same_bits

GOLD = golden_util.load()
BINBY = sorted(k for k in GOLD if not k.startswith(("set_", "hash64")))
SETS = sorted(k for k in GOLD if k.startswith("set_"))


@pytest.mark.parametrize("name", BINBY)
def test_oracle_matches_golden_binby(name, oracle):
    binners, aggs, n, expected = golden_util.binby_case(GOLD[name])
    got = oracle.binby(binners, aggs, n)
    for a, w, g in zip(aggs, expected, got):
        assert same(w, g), (name, a["op"])


def test_golden_kats_are_the_reference_test_vectors():
    # /root/reference/tests/agg_test.py:150-158 and :171-180
    assert GOLD["kat_count_1d"]["a0_result"].tolist() == [0, 2, 1, 1, 0, 0, 1, 1]
    assert GOLD["kat_count_1d_ordinal"]["a0_result"].tolist() == [1, 1, 0, 0, 1, 3, 0]


@pytest.mark.parametrize("name", SETS)
def test_oracle_matches_golden_sets(name, oracle):
    c = GOLD[name]
    dtype, nmaps = name.split("_")[1], int(name.split("_")[2])
    s = oracle.OrderedSet(dtype, nmaps)
    vals, mi = s.update(c["keys"], c["mask"], 0, True)
    assert np.array_equal(vals, c["values"]) and np.array_equal(mi, c["map_index"])
    assert np.array_equal(s.key_array(), c["key_array"], equal_nan=True)
    assert s.offsets() == c["offsets"].tolist()
    mo = s.map_ordinal(c["keys"])
    assert mo.dtype == c["map_ordinal"].dtype and np.array_equal(mo, c["map_ordinal"])
    assert [s.null_index, s.nan_index, s.null_count, s.nan_count] == c["null_nan"].tolist()


def test_hash64_golden(oracle):
    for i, o in zip(GOLD["hash64"]["in"], GOLD["hash64"]["out"]):
        assert oracle.hash64(int(i)) == int(o)
    assert oracle.hash64(1) == 6238072747940578789  # SURVEY.md 8c pin


@pytest.mark.parametrize("seed", range(12))
def test_oracle_matches_compiled_reference_random(seed, oracle, ref):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(1, 5000))
    binners, aggs = random_case(rng, n)
    want = ref.binby(binners, aggs, n)
    got = oracle.binby(binners, aggs, n)
    for a, w, g in zip(aggs, want, got):
        assert same_bits(np.asarray(w) if not np.ma.isMaskedArray(w) else w, g), (a["op"], None if a["data"] is None else a["data"].dtype)


@pytest.mark.parametrize("seed", range(40))
def test_oracle_matches_compiled_reference_edges(seed, oracle, ref):
    """the edge-value corpus (random_case(edges=True): integer limits, uint64 >= 2^63, +-0.0, +-inf, NaN payloads, subnormals,
    overflowing powers, keys on bin edges, byte-swapped twins, moments 0..8, nunique), bit for bit"""
    rng = np.random.default_rng(7000 + seed)
    n = int(rng.integers(1, 3000))
    binners, aggs = random_case(rng, n, edges=True)
    want = ref.binby(binners, aggs, n)
    got = oracle.binby(binners, aggs, n)
    for a, w, g in zip(aggs, want, got):
        assert same_bits(np.asarray(w) if not np.ma.isMaskedArray(w) else w, g), (a["op"], a.get("moment"), None if a["data"] is None else a["data"].dtype)


EDGES = golden_util.load_edges()


@pytest.mark.parametrize("name", sorted(EDGES))
def test_oracle_matches_golden_edges(name, oracle):
    """tests/golden/edges_golden.npz: edge-value cases and single-cell known answers from the compiled reference"""
    binners, aggs, n, expected = golden_util.binby_case(EDGES[name])
    got = oracle.binby(binners, aggs, n)
    for a, w, g in zip(aggs, expected, got):
        assert same_bits(w, g), (name, a["op"])


def test_golden_edges_known_answers():
    """the values the compiled reference gives for the cases where the device's rule is documented (DESIGN §3)"""
    imin = np.iinfo(np.int64).min
    assert EDGES["kat_moment3_int64_out_of_range"]["a0_result"].ravel()[2] == imin
    assert EDGES["kat_moment3_uint64_out_of_range"]["a0_result"].ravel()[2] == 0
    # 30000^4 + 30001^4 + 29999^4 + 1 = 2430000010800000003 exactly; the reference rounds its running sum through double
    assert EDGES["kat_moment4_past_2p53"]["a0_result"].ravel()[2] == 2430000010800000000
    r = EDGES["kat_minmax_signed_zeros"]
    assert [np.signbit(r["a0_result"].ravel()[2]), np.signbit(r["a1_result"].ravel()[2])] == [True, True]


def test_exact_sum_check_is_not_vacuous(oracle):
    """helpers.float_sum_ok (the recursive-summation bound of the GPU tests) accepts the oracle and rejects a wrong cancelling sum"""
    from helpers import float_sum_ok
    v = np.array([1e16, 1.0, -1e16, 1.0])
    b = [oracle.scalar(np.full(4, 0.5), 0, 1, 1)]
    a = oracle.agg("sum", v)
    w = oracle.binby(b, [a], 4)[0]
    assert float_sum_ok(b, a, 4, w) is None
    bad = w.copy()
    bad.ravel()[2] = 100.0  # the bound here is gamma_4 * 2e16 ~ 9
    assert float_sum_ok(b, a, 4, bad) is not None


def test_oracle_first_mask_quirk_matches_reference(oracle, ref):
    """AggFirst indexes its mask inside the 1024-row block without the block offset (src/agg_first.cpp:131);
    the oracle restates that, so both agree even past 1024 rows."""
    rng = np.random.default_rng(77)
    n = 3000
    x = rng.uniform(0, 4, n)
    v = rng.normal(0, 1, n)
    o = rng.integers(0, 100, n).astype("i8")
    m = (rng.random(n) < 0.6).astype("u1")
    b = [oracle.scalar(x, 0, 4, 4)]
    a = [oracle.agg("first", v, m, order=o), oracle.agg("last", v, m, order=o)]
    for w, g in zip(ref.binby(b, a, n), oracle.binby(b, a, n)):
        assert same(w, g)


@pytest.mark.parametrize("nthreads", [1, 4])
def test_reference_chunk_loop_is_thread_invariant_for_counts(nthreads, oracle, ref):
    """the restated executor loop (1M-row chunks, per-thread grids folded in get_result) gives the same exact counts"""
    rng = np.random.default_rng(5)
    n = 300_000
    x = rng.normal(0, 1, n).astype("f4")
    y = rng.normal(0, 1, n).astype("f4")
    b = [oracle.scalar(x, -3, 3, 64), oracle.scalar(y, -3, 3, 64)]
    a = [oracle.agg("count")]
    want = oracle.binby(b, a, n)[0]
    got = ref.RefBinby(b, a, nthreads).run(n, chunk=50_000)[0]
    assert np.array_equal(want, np.asarray(got))


# ---- limits pre-pass (df.minmax): SURVEY.md section 8f row 1 ------------------------------------------------------------------
MINMAX = golden_util.load_minmax()


@pytest.mark.parametrize("name", sorted(MINMAX))
def test_oracle_minmax_matches_golden(name, oracle):
    """oracle.minmax (orc_minmax) against vaexfast.statisticNd OP_MIN_MAX of the compiled reference: all 11 dtypes, masked,
    byte-swapped, NaN / inf, integers beyond 2^24 / 2^53 (rounded by the reference's float casts), empty and all-NaN columns."""
    data, raw, result = MINMAX[name]
    assert np.array_equal(oracle.minmax(data, raw=True), raw, equal_nan=True)
    got = oracle.minmax(data)
    assert got.dtype == result.dtype and np.array_equal(got, result, equal_nan=True)


def test_minmax_float_cast_quirk_is_in_the_golden_vectors():
    # int32 max - 1 = 2147483646 is not a float32: the reference reports 2147483648.0 in its grid (vaex/cpu.py:519-531)
    _, raw, _ = MINMAX["int32"]
    assert raw[1] == 2147483648.0
    _, raw, _ = MINMAX["int64"]
    assert raw[1] == 9223372036854775808.0  # int64 goes through float64


@pytest.mark.parametrize("seed", range(6))
def test_oracle_minmax_matches_compiled_reference_random(seed, oracle, ref):
    rng = np.random.default_rng(4000 + seed)
    n = int(rng.integers(1, 20000))
    for dt in ("f8", "f4", "i8", "i4", "i2", "i1", "u8", "u4", "u2", "u1", "?", ">f8", ">i4", ">u2"):
        d = np.dtype(dt)
        if d.kind == "f":
            v = (rng.standard_normal(n) * 10.0 ** int(rng.integers(-3, 6))).astype(d)
            v[rng.random(n) < 0.2] = np.nan
        elif d.kind == "b":
            v = rng.integers(0, 2, n).astype(d)
        else:
            info = np.iinfo(d)
            v = rng.integers(info.min, info.max, n, dtype=np.int64 if d.kind == "i" else np.uint64, endpoint=True).astype(d)
        for col in (v, np.ma.array(v, mask=rng.random(n) < 0.5)):
            assert np.array_equal(oracle.minmax(col, raw=True), ref.minmax(col, raw=True), equal_nan=True), dt


# ---- string key sets (SURVEY.md section 8f row 3) ----------------------------------------------------------------------------------
STRINGS = golden_util.load_strings()


def test_string_hash_known_answers(oracle):
    """std::hash<string_view> of the reference build = libstdc++'s 64-bit Murmur-2 (src/hash.hpp:59-86)"""
    c = STRINGS["strhash"]
    keys = [bytes(c["bytes"][c["offsets"][i]:c["offsets"][i + 1]]) for i in range(len(c["offsets"]) - 1)]
    assert [oracle.string_hash(k) for k in keys] == [int(h) for h in c["hash"]]


@pytest.mark.parametrize("name", sorted(k for k in STRINGS if k.startswith("strset_")))
def test_oracle_string_set_matches_golden(name, oracle):
    c = STRINGS[name]
    s = oracle.StringOrderedSet(int(name.split("_")[1]))
    for k in range(int(c["ncalls"])):
        strs = golden_util.unpack_strings(c[f"c{k}_offsets"], c[f"c{k}_bytes"], c[f"c{k}_mask"])
        vals, mi = s.update(strs, 0, True)
        assert np.array_equal(vals, c[f"c{k}_values"]) and np.array_equal(mi, c[f"c{k}_map_index"])
    assert s.keys() == golden_util.unpack_strings(c["key_offsets"], c["key_bytes"], c["key_nulls"])
    assert s.offsets() == c["shard_offsets"].tolist()
    probe = golden_util.unpack_strings(c["probe_offsets"], c["probe_bytes"], c["probe_mask"])
    assert np.array_equal(s.map_ordinal(probe), c["probe_ordinals"])
    assert [len(s), s.null_count, s.null_index] == c["info"].tolist()


def test_agg_list_restatement_matches_the_compiled_reference_vectors():
    """oracle.agg_list (src/agg_list.cpp restated, incl. the mask-without-block-offset quirk) against the vectors the compiled
    reference's AggList_<dtype>_int64 produced (tests/golden/make_golden_agglist.py): 5 dtypes x plain / masked x dropnan x dropnull,
    fed in two calls of 1777 and 2223 rows (so the 1024-row blocks and the call boundary both matter)."""
    import golden_util
    from oracle import oracle as O
    g = golden_util.load_agglist()
    x, n = g["x"], len(g["x"])
    cells = O.flat_indices([O.ordinal(x, g["ncat"], 0)], n)[0].astype(np.int64)
    assert len(g["cases"]) == 40
    for name, c in g["cases"].items():
        off, vals, _, _ = O.agg_list(cells, c["v"], c["valid"] if c["masked"] else None, len(c["offsets"]) - 1, c["dropnan"], c["dropnull"],
                                     calls=[(0, g["cut"]), (g["cut"], n)])
        assert np.array_equal(off, c["offsets"]), name
        assert np.array_equal(vals, c["values"], equal_nan=True), name
