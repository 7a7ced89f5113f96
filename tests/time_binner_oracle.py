"""The time binner's integer steps (csrc/device_utils.cuh time_steps / time_period / time_bin) restated in numpy int64: floor division,
numpy's week epoch, days <-> proleptic Gregorian months and the `every` step.  tests/test_time_binner_cpu.py holds it equal to numpy's
own astype('M8[R]'); the GPU tests hold the device to it."""
import numpy as np

UNITS = ["Y", "M", "W", "D", "h", "m", "s", "ms", "us", "ns"]
NS = {"W": 604800 * 10 ** 9, "D": 86400 * 10 ** 9, "h": 3600 * 10 ** 9, "m": 60 * 10 ** 9, "s": 10 ** 9, "ms": 10 ** 6, "us": 10 ** 3, "ns": 1}
NAT = np.iinfo(np.int64).min


def _fdiv(n, d):
    """floor(n / d) of int64 n by a positive d, as the device's sign trick computes it: ~((~n) // d) for n < 0"""
    n = np.asarray(n, dtype=np.int64)
    neg = n < 0
    u = np.where(neg, ~n, n).astype(np.uint64) // np.uint64(d)
    return np.where(neg, ~u.astype(np.int64), u.astype(np.int64))


def _mul(n, m):
    """n * m with int64 wrap-around"""
    return (np.asarray(n, dtype=np.int64).astype(np.uint64) * np.uint64(m)).astype(np.int64)


def steps(unit, res):
    """time_steps: (civil_in, civil_out, years, mul, div)"""
    civil_u, civil_r = unit in ("Y", "M"), res in ("Y", "M")
    if civil_u and civil_r:
        frm, to = (12 if unit == "Y" else 1), (12 if res == "Y" else 1)
        civil_in = civil_out = years = False
    else:
        civil_in, civil_out = civil_u, (not civil_u) and civil_r
        years = (civil_in and unit == "Y") or (civil_out and res == "Y")
        frm, to = NS["D" if civil_u else unit], NS["D" if civil_r else res]
    return civil_in, civil_out, years, (1 if to >= frm else frm // to), (to // frm if to >= frm else 1)


def days_from_months(months):
    months = np.asarray(months, dtype=np.int64)
    yq = _fdiv(months, 12)
    m = months - yq * 12
    y = yq + 1970 - (m < 2)
    era = _fdiv(y, 400)
    yoe = y - era * 400
    mp = np.where(m < 2, m + 10, m - 2)
    doe = yoe * 365 + yoe // 4 - yoe // 100 + (153 * mp + 2) // 5
    return era * 146097 + doe - 719468


def months_from_days(days, years):
    days = np.asarray(days, dtype=np.int64)
    q = _fdiv(days, 146097)
    z = days - q * 146097 + 719468
    era = q + z // 146097
    doe = z % 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    y = era * 400 + yoe + (mp >= 10) - 1970
    return y if years else y * 12 + np.where(mp < 10, mp + 2, mp - 10)


def period(t, unit, res):
    """time_period: the period of resolution `res` of the int64 ticks t of `unit` (NaT not special-cased)"""
    civil_in, civil_out, years, mul, div = steps(unit, res)
    t = np.asarray(t, dtype=np.int64)
    with np.errstate(over="ignore"):
        if civil_in:
            t = days_from_months(_mul(t, 12) if years else t)
        p = _fdiv(_mul(t, mul), div)
        if civil_out:
            p = months_from_days(p, years)
    return p


def bins(t, unit, res, begin, every, n, masked=None):
    """time_bin + ordinal_index: the cell of every row, n for NaT, masked and out-of-range rows"""
    t = np.asarray(t, dtype=np.int64)
    with np.errstate(over="ignore"):
        b = _fdiv((period(t, unit, res).astype(np.uint64) - np.uint64(begin & 0xFFFFFFFFFFFFFFFF)).astype(np.int64), every)
    null = (t == NAT) | (b < 0) | (b >= n)
    if masked is not None:
        null |= np.asarray(masked, bool)
    return np.where(null, n, b)
