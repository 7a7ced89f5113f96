"""AggList_string_int64 without a GPU: the oracle's restatement against the compiled reference's golden vectors and (where it is
built) against the compiled reference itself, the mirror's string class names, and the class lookup of string dtypes."""
import importlib
import random
import sys
import types

import numpy as np
import pytest

import agglist_string_cases as cases
from oracle.agglist_string import agg_list_string


def _expected(oracle, setup, case):
    cells, ncells = cases.flat_cells(setup)
    return agg_list_string(cells, cases.strings_of(setup), ncells, dropnan=case["dropnan"], dropnull=case["dropnull"],
                           mask=setup["valid"] if case["masked"] else None)


@pytest.mark.parametrize("setup_name", cases.SETUPS)
def test_oracle_matches_golden_agglist_string(setup_name, oracle):
    setup = cases.load()[setup_name]
    assert len(setup["cases"]) == 8
    for name, case in setup["cases"].items():
        lo, so, by, va = _expected(oracle, setup, case)
        assert np.array_equal(lo, case["list_offsets"]), name
        assert np.array_equal(so, case["str_offsets"]), name
        assert np.array_equal(by, case["str_bytes"]), name
        assert np.array_equal(va, case["str_valid"]), name


def test_golden_agglist_string_covers_the_cases():
    g = cases.load()
    setup = g["ord"]
    strs = [s for s in cases.strings_of(setup) if s is not None]
    assert "" in strs and any(len(s.encode()) > 4096 for s in strs) and any(len(s.encode()) > 64 for s in strs)
    assert any(len(s.encode()) != len(s) for s in strs)  # multi-byte UTF-8
    assert setup["nulls"].any() and not setup["valid"].all()
    assert all(i1 % 1024 for _, i1 in setup["calls"][:-1]) and len(setup["calls"]) == 3
    # the data mask is never read: masked and plain results are the same
    for d in ("dropnan0_dropnull0", "dropnan1_dropnull1"):
        assert np.array_equal(setup["cases"]["masked_" + d]["str_bytes"], setup["cases"]["plain_" + d]["str_bytes"])
    # dropnull=False keeps the nulls: they show up as invalid elements
    assert (setup["cases"]["plain_dropnan0_dropnull0"]["str_valid"] == 0).any()
    assert (setup["cases"]["plain_dropnan0_dropnull1"]["str_valid"] == 1).all()
    one = g["one_cell"]["cases"]["plain_dropnan0_dropnull0"]["list_offsets"]
    assert (np.diff(one) > 0).sum() == 1
    sparse = g["sparse"]["cases"]["plain_dropnan0_dropnull0"]["list_offsets"]
    assert (np.diff(sparse) == 0).sum() > len(sparse) // 2


def _ref_string_list(ref):
    """the compiled reference's AggList_string_int64 fed through oracle/ref_strlist_shim.cpp, with vaex.arrow.convert stubbed"""
    vaex = types.ModuleType("vaex")
    arrow = types.ModuleType("vaex.arrow")
    convert = types.ModuleType("vaex.arrow.convert")
    convert.list_from_arrays = lambda offsets, values: (np.array(offsets), values)
    vaex.arrow, arrow.convert = arrow, convert
    saved = {k: sys.modules.get(k) for k in ("vaex", "vaex.arrow", "vaex.arrow.convert")}
    sys.modules.update({"vaex": vaex, "vaex.arrow": arrow, "vaex.arrow.convert": convert})
    sys.path.insert(0, ref._REF)
    try:
        shim = importlib.import_module("strlist_shim")
    except ImportError:
        pytest.skip("oracle/_ref/strlist_shim not built (make -C oracle -f strlist_shim.mk)")
    finally:
        sys.path.remove(ref._REF)
    return shim, saved


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_compiled_reference_random(seed, oracle, ref):
    superagg, _ = ref.modules()
    shim, saved = _ref_string_list(ref)
    try:
        rnd = random.Random(seed)
        rng = np.random.default_rng(seed)
        n = int(rng.integers(1, 5000))
        ncat = int(rng.integers(1, 40))
        x = rng.integers(-2, ncat + 2, n).astype("i8")
        words = ["", "a", "äß€", "x" * 70] + ["".join(rnd.choice("abc😀") for _ in range(rnd.randint(1, 20))) for _ in range(50)]
        strs = [None if rnd.random() < 0.15 else rnd.choice(words) for _ in range(n)]
        off, by, nulls = ref.pack_strings(strs)
        cuts = sorted(set(int(c) for c in rng.integers(1, n, 2))) if n > 2 else []
        calls = list(zip([0] + cuts, cuts + [n]))
        dropnull = bool(seed & 1)
        b = superagg.BinnerOrdinal_int64(1, "x", ncat, 0, False, False)
        g = superagg.Grid([b])
        a = superagg.AggList_string_int64(g, 1, 1, False, dropnull)
        keep = []
        for i1, i2 in calls:
            xs = np.ascontiguousarray(x[i1:i2])
            sl = shim.make(np.ascontiguousarray(off[i1:i2 + 1] - off[i1]), np.ascontiguousarray(by[off[i1]:off[i2]]), np.ascontiguousarray(nulls[i1:i2]))
            keep += [xs, sl]
            b.set_data(0, xs)
            a.set_data(0, sl, 0)
            g.bin(0, [a], i2 - i1)
        list_offsets, res = a.get_result()
        got = (np.asarray(list_offsets, np.int64),) + tuple(np.asarray(v) for v in shim.buffers(res))
        cells = oracle.flat_indices([oracle.ordinal(x, ncat, 0)], n)[0].astype(np.int64)
        want = agg_list_string(cells, strs, ncat + 2, dropnull=dropnull)
        for gv, wv in zip(got, want):
            assert np.array_equal(gv, wv)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_every_reference_string_aggregator_resolves_in_the_mirror(ref):
    superagg, _ = ref.modules()
    from vaex_b200 import superagg as mine
    # the reference's experimental BinnerHash_string stays out, like the numeric BinnerHash_* (see vaex_b200.superagg._BinnerHash)
    want = [n for n in dir(superagg) if n.startswith("Agg") and "_string" in n]
    assert "AggList_string_int64" in want
    assert not [n for n in want if not hasattr(mine, n)]


def test_find_type_from_dtype_resolves_string_classes():
    from vaex_b200 import agg, superagg
    obj, i64 = np.dtype("O"), np.dtype("int64")
    assert agg.find_type_from_dtype(superagg, "AggList_", obj, i64) is superagg.AggList_string_int64
    assert agg.find_type_from_dtype(superagg, "AggList_", np.dtype("U5"), i64) is superagg.AggList_string_int64
    assert agg.find_type_from_dtype(superagg, "AggCount_", obj) is superagg.AggCount_string
    assert agg.find_type_from_dtype(superagg, "AggNUnique_", obj) is superagg.AggNUnique_string
    assert agg.find_type_from_dtype(superagg, "AggList_", np.dtype("f8"), i64) is superagg.AggList_float64_int64
    with pytest.raises(ValueError, match="strings are not supported"):
        agg.find_type_from_dtype(superagg, "AggSum_", obj)


def test_list_string_descriptor_picks_the_string_aggregator():
    from vaex_b200 import agg, superagg
    d = agg.list("s", dropmissing=True)
    d._prepare_types({"s": np.dtype("O")})
    grid = superagg.Grid([superagg.BinnerOrdinal_int64(1, "k", 3)])
    try:
        op = d._create_operation(grid, 1)
    except RuntimeError as e:  # no GPU here: the aggregator object cannot be created, but the class lookup happened first
        assert "sm_90" in str(e) or "device" in str(e) or "CUDA" in str(e)
        return
    assert isinstance(op, superagg.AggList_string_int64)
