"""The time binner's integer steps (time_binner_oracle.py, the device's arithmetic in numpy) against numpy's own astype('M8[R]') for every
(unit, resolution) pair, the host's exact period check, and the reference's groupby binner cases against a numpy groupby."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import groupby_binner_cases as GC  # noqa: E402
import time_binner_oracle as TB  # noqa: E402

from vaex_b200 import groupby as G  # noqa: E402

I64 = np.iinfo(np.int64)
DATES = ["1600-02-29", "1899-12-31", "1900-02-28", "1900-03-01", "1969-12-31T23:59:59.999999999", "1970-01-01", "1970-01-04", "1970-01-08",
         "1999-12-31T23:59:59", "2000-02-29", "2000-03-01", "2100-02-28", "2100-03-01", "2262-04-11", "1677-09-22"]


def corpus(unit):
    """ticks of `unit`: small values, the dates above, period boundaries of every coarser resolution +- 1 tick, the int64 extremes"""
    v = [I64.min + 1, I64.max, -2 ** 62, 2 ** 62, -2 ** 53, 2 ** 53] + list(range(-1000, 1001))
    for d in DATES:
        v.append(int(np.datetime64(d).astype(f"M8[{unit}]").astype(np.int64)))
    for res in TB.UNITS[:TB.UNITS.index(unit)]:
        starts = np.arange(-3000, 3000, 7 if res not in "YM" else 1).astype(f"M8[{res}]").astype(f"M8[{unit}]").astype(np.int64)
        for s in starts:
            v += [int(s) - 1, int(s), int(s) + 1]
    v = np.unique(np.array(v, dtype=np.int64))
    return v[v != TB.NAT]


@pytest.mark.parametrize("unit", TB.UNITS)
@pytest.mark.parametrize("res", TB.UNITS)
def test_period_equals_numpy(unit, res):
    """where numpy's conversion does not overflow (the exact Python result fits int64), the oracle gives numpy's period; the host
    check (groupby.period) gives it too"""
    t = corpus(unit)
    exact = np.array([G.period(int(x), unit, res) for x in t], dtype=object)
    fits = np.array([I64.min < e <= I64.max for e in exact])
    with np.errstate(over="ignore"):
        want = t.astype(f"M8[{unit}]").astype(f"M8[{res}]").astype(np.int64)
    ok = fits & (want == np.array([e if f else 0 for e, f in zip(exact, fits)], dtype=object))
    # numpy is exact wherever the result fits, except for year/month arithmetic at the extremes of the int64 range
    assert ok.sum() >= fits.sum() - 8, (unit, res, t[fits & ~ok][:5])
    got = TB.period(t[ok], unit, res)
    np.testing.assert_array_equal(got, want[ok])


@pytest.mark.parametrize("unit", ["D", "s", "ns", "M", "Y", "W"])
@pytest.mark.parametrize("res", ["Y", "M", "W", "D", "h"])
@pytest.mark.parametrize("every", [1, 3, 7])
def test_bins_equal_reference_expression(unit, res, every):
    """the reference's BinnerTime expression (t.astype('M8[R]') - begin).astype('int') // every -> BinnerOrdinal(N): NaT and bins
    outside [0, N) go to the null cell N"""
    rng = np.random.default_rng(TB.UNITS.index(unit) * 100 + TB.UNITS.index(res) * 10 + every)
    lo = int(np.datetime64("1890-01-01").astype(f"M8[{unit}]").astype(np.int64))
    hi = int(np.datetime64("2110-01-01").astype(f"M8[{unit}]").astype(np.int64))
    t = rng.integers(lo, hi, 5000).astype(f"M8[{unit}]")
    t[::97] = np.datetime64("NaT")
    valid = t[~np.isnat(t)]
    tmin, tmax = valid[len(valid) // 4:].min(), valid.max()  # a begin inside the data: rows before it are out of range
    begin = tmin.astype(f"M8[{res}]")
    n = ((tmax.astype(f"M8[{res}]") - begin).astype(int) + every) // every
    with np.errstate(invalid="ignore"):
        codes = (t.astype(f"M8[{res}]") - begin).astype("int64") // every
    want = np.where((codes < 0) | (codes >= n), n, codes)
    got = TB.bins(t.astype(np.int64), unit, res, int(begin.astype(np.int64)), every, n)
    np.testing.assert_array_equal(got, want)


def test_bins_null_and_masked():
    t = np.array([0, TB.NAT, 5, 6], dtype=np.int64)
    np.testing.assert_array_equal(TB.bins(t, "D", "D", 0, 1, 7, masked=[0, 0, 1, 0]), [0, 7, 7, 6])


def test_period_host_check_overflow():
    """numpy wraps a finer resolution silently; the exact period shows the overflow"""
    t = int(np.datetime64("2300-01-01", "D").astype(np.int64))
    assert np.datetime64("2300-01-01", "D").astype("M8[ns]").astype(np.int64) != t * 86400 * 10 ** 9
    assert G.period(t, "D", "ns") > I64.max
    assert G.period(-1, "s", "m") == -1  # np.datetime64(-1, 's') -> 1969-12-31T23:59


@pytest.mark.parametrize("case", GC.CASES, ids=[c[0] for c in GC.CASES])
def test_reference_case_in_numpy(case):
    name, columns, keys, agg, expected, kwargs = case
    got = GC.numpy_groupby(columns, keys, agg)
    if "__len__" in expected:
        assert len(got["values"]) == expected["__len__"] and sum(got["values"]) == expected["__sum__"]
        return
    labels = [k if isinstance(k, str) else k[1] for k in keys]
    value = [k for k in expected if not k.startswith("__")][-1]  # the aggregate is the last output of a case
    for i, label in enumerate(labels):
        if label in expected and label != value:
            got_keys = [k[i] for k in got["keys"]]
            assert got_keys == (pytest.approx(expected[label]) if isinstance(expected[label][0], float) else expected[label])
    if "__first_list__" in expected:
        assert set(got["values"][0]) == expected["__first_list__"]
    else:
        assert got["values"] == expected[value]
