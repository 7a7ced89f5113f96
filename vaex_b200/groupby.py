"""vaex's groupby binners (vaex/groupby.py:35-224) for Frame.groupby: ``Binner`` (value ranges), ``BinnerInteger`` (integer ranges with a
null group) and ``BinnerTime`` (calendar periods).  Each one is a spec of a device binner plus the keys of its cells:
  * Binner         -> the scalar binner (BinnerScalar), keys = the bin centers, cells [2:-1];
  * BinnerInteger  -> the ordinal binner (BinnerOrdinal with min_value / invert), keys = a masked array whose last key is the null
                      group, cells [0:-1] (or [0:-2] with dropmissing);
  * BinnerTime     -> the time binner (B200_BINNER_TIME): the period of every row is computed in the binning kernel from the column's
                      raw ticks, as numpy's astype('M8[R]') computes it, keys = datetime64[R], cells [0:-2].
Frame.__getitem__ returns raw columns, so every binner takes its expression as a string plus ``df=``."""
import numpy as np

from . import _lib

__all__ = ["Binner", "BinnerInteger", "BinnerTime"]

_INT64_MIN, _INT64_MAX = -2 ** 63, 2 ** 63 - 1
_MAX_PERIODS = 2 ** 31  # the keys are a host array of N datetimes and every aggregator a grid of N + 2 cells
# nanoseconds per tick of the linear units (W .. ns); Y and M are calendar units
_NS = {"W": 604800 * 10 ** 9, "D": 86400 * 10 ** 9, "h": 3600 * 10 ** 9, "m": 60 * 10 ** 9, "s": 10 ** 9, "ms": 10 ** 6, "us": 10 ** 3, "ns": 1}


class BinnerBase:
    """a grouper whose cells are fixed before the pass: `spec(df)` is its device binner, `bin_values` the keys of the cells
    [start, start + len(bin_values)) of its grid axis"""
    dense = False
    start = 0

    def _resolve(self, expression, df, label):
        if df is None:
            raise TypeError(f"{type(self).__name__} needs df=: Frame columns are plain arrays, the binner takes the expression's frame")
        self.df = df
        self.expression = str(expression)
        self.label = label or self.expression

    def __repr__(self):
        return f"{type(self).__name__}({self.expression!r})"


class Binner(BinnerBase):
    """vaex.groupby.Binner: groups by `bins` equal ranges of [vmin, vmax); keys are the bin centers"""
    start = 2

    def __init__(self, expression, vmin, vmax, bins, df=None, label=None):
        self._resolve(expression, df, label)
        self.vmin, self.vmax, self.N = vmin, vmax, int(bins)
        self.cells = self.N + 3
        self.bin_values = df.bin_centers(self.expression, (vmin, vmax), self.N)

    def spec(self, df):
        from .frame import _scalar_spec
        return _scalar_spec(self.expression, _lib.dtype_of(df.columns[self.expression]), self.N, (self.vmin, self.vmax))


class BinnerInteger(BinnerBase):
    """vaex.groupby.BinnerInteger: every integer of [min_value, max_value] is a group (bool, int8 and uint8 take their full range),
    plus a null group that also takes the values outside that range; sort=True, ascending=False orders the groups descending"""

    def __init__(self, expression, label=None, dropmissing=False, min_value=None, max_value=None, dense=False, sort=False, ascending=True, df=None):
        self._resolve(expression, df, label)
        self.dtype = df._with_columns([self.expression]).dtypes()[self.expression]
        self.min_value = 0
        self.dropmissing = dropmissing
        self.dense = dense
        descending = sort and not ascending

        def make_array_with_null(vmin, vmax, dtype="int64"):
            values = np.arange(vmax - 1, vmin - 2, -1, dtype=dtype) if descending else np.arange(vmin, vmax + 1, dtype=dtype)
            mask = np.zeros(values.shape, dtype="?")
            mask[len(values) - 1] = 1
            values[len(values) - 1] = 0
            return np.ma.array(values, mask=mask, shrink=False)

        if self.dtype == np.dtype("bool"):
            # the reference does not reverse these keys when it inverts the cells (vaex/groupby.py:159-163): kept
            self.bin_values = np.ma.array([False, True, False], mask=[False, False, True], shrink=False)
            self.N = 2
        elif self.dtype == np.dtype("uint8"):
            self.bin_values = make_array_with_null(0, 256)
            self.N = 256
        elif self.dtype == np.dtype("int8"):
            self.min_value = -128
            self.bin_values = make_array_with_null(-128, 128)
            self.N = 256
        elif min_value is not None and max_value is not None:
            self.min_value = min_value
            self.N = int(max_value - min_value + 1)
            self.bin_values = make_array_with_null(min_value, max_value + 1)
        else:
            raise TypeError(f"Only boolean, int8 and uint8 are supported, not {self.dtype}, or private min_value and max_value")
        if self.dropmissing:
            self.bin_values = self.bin_values[:-1]
        self.invert = descending
        self.cells = self.N + 2

    def spec(self, df):
        return {"binner-type": "ordinal", "expression": self.expression, "dtype": _lib.dtype_of(df.columns[self.expression]).str, "count": self.N,
                "minimum": int(self.min_value), "invert": bool(self.invert)}


class BinnerTime(BinnerBase):
    """vaex.groupby.BinnerTime: groups a datetime64 column by periods of `every` units of `resolution` (Y M W D h m s ms us ns), from
    the first period present in the rows of `df` (its filter applies) to the last; every period in between is a cell, and the
    groups with rows are returned.  Weeks start on Thursday (numpy's week 0 is 1970-01-01); per_quarter is three months from the
    first month present."""

    def __init__(self, expression, resolution="W", df=None, every=1):
        self._resolve(expression, df, None)
        self.resolution, self.every = resolution, int(every)
        if resolution not in _lib.TIME_UNITS:
            raise ValueError(f"resolution must be one of {_lib.TIME_UNITS}, not {resolution!r}")
        if self.every < 1:
            raise ValueError(f"every must be at least 1, not {every}")
        col = df.columns.get(self.expression)
        dtype = None if col is None else _lib.dtype_of(col)
        if dtype is None or dtype.kind != "M":
            raise TypeError(f"BinnerTime needs a datetime64 column of the frame, not {self.expression!r}" + ("" if dtype is None else f" of dtype {dtype}"))
        self.unit, step = np.datetime_data(dtype)
        if self.unit not in _lib.TIME_UNITS or step != 1:
            raise ValueError(f"BinnerTime supports the units {_lib.TIME_UNITS} without a multiplier, not {dtype}")
        self.dtype = dtype
        self.tmin, self.tmax = _limits(df, self.expression, col, dtype)
        begin, end = (period(int(t.astype(np.int64)), self.unit, resolution) for t in (self.tmin, self.tmax))
        for p, t in ((begin, self.tmin), (end, self.tmax)):
            if not _INT64_MIN < p <= _INT64_MAX:
                raise ValueError(f"{t} has no datetime64[{resolution}] value: {p} overflows int64 (numpy would wrap it)")
        self.begin = begin
        self.N = (end - begin + self.every) // self.every
        if self.N > _MAX_PERIODS:
            raise ValueError(f"{self.tmin} .. {self.tmax} spans {self.N} periods of {self.every} {resolution}: more cells than one grid holds "
                             f"({_MAX_PERIODS})")
        self.cells = self.N + 2
        self.bin_values = np.arange(np.datetime64(begin, resolution), np.datetime64(end, resolution) + 1, self.every)

    def spec(self, df):
        return {"binner-type": "time", "expression": self.expression, "dtype": _lib.dtype_of(df.columns[self.expression]).str, "resolution": self.resolution,
                "begin": self.begin, "count": self.N, "every": self.every}

    @classmethod
    def per_day(cls, expression, df=None):
        return cls(expression, "D", df)

    @classmethod
    def per_week(cls, expression, df=None):
        return cls(expression, "W", df)

    @classmethod
    def per_month(cls, expression, df=None):
        return cls(expression, "M", df)

    @classmethod
    def per_quarter(cls, expression, df=None, every=1):
        return cls(expression, "M", df, every=3 * every)

    @classmethod
    def per_year(cls, expression, df=None):
        return cls(expression, "Y", df)


def _floordiv_days_to_civil(days):
    """days since 1970-01-01 -> (year, month 1..12), proleptic Gregorian, exact for any Python int"""
    z = days + 719468
    era, doe = divmod(z, 146097)
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    m = mp + 3 if mp < 10 else mp - 9
    return era * 400 + yoe + (m <= 2), m


def _civil_to_days(y, m):
    """the first day of month m (1..12) of year y, in days since 1970-01-01"""
    y -= m <= 2
    era, yoe = divmod(y, 400)
    mp = (m + 9) % 12
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + (153 * mp + 2) // 5 - 719468


def period(t, unit, resolution):
    """the exact period of resolution R of the tick t of unit U, as a Python int (numpy's astype('M8[R]') without its int64
    wrap-around): the host check that the device's int64 steps do not overflow"""
    civil_u, civil_r = unit in "YM", resolution in "YM"
    if civil_u:
        y, m = divmod(t * 12 if unit == "Y" else t, 12)
        if civil_r:
            return (y * 12 + m) // (12 if resolution == "Y" else 1)
        t, unit = _civil_to_days(1970 + y, m + 1), "D"
    if civil_r:
        y, m = _floordiv_days_to_civil(t * _NS[unit] // _NS["D"])
        return y - 1970 if resolution == "Y" else (y - 1970) * 12 + m - 1
    return t * _NS[unit] // _NS[resolution]


def _limits(df, expression, col, dtype):
    """(tmin, tmax) of the column over the rows of df, as the reference's BinnerTime takes them (vaex/groupby.py:100): df.minmax, the
    legacy statistic of class float32 for a datetime block (vaex/cpu.py:526-540), cast back to the column's dtype
    (vaex/dataframe.py:1524-1528).  NaT is left out: the reference counts it as -2^63 and its limits break (DESIGN.md section 3)."""
    ticks = "__ticks_" + expression
    data, _ = _lib.split_mask(col)
    view = _lib.int64_view(data if _lib.is_device(data) else np.asarray(data).astype(dtype.newbyteorder("=")))
    f = df._derive(dict(df.columns))
    f.columns[ticks] = view
    res = f.minmax(expression, selection=f"{ticks} != {_INT64_MIN}")
    if not np.all(np.isfinite(res)):
        raise ValueError(f"BinnerTime: {expression!r} has no value that is not NaT in the frame's rows")
    return tuple(res.astype(dtype.newbyteorder("=")))
