"""The cases behind tests/golden/statistic_golden.npz: known answers of the legacy statistics (statisticNd) plus a fixed set of random
problems from tests/statistic_cases.py.  Each case is a dict of statistic_oracle.process keyword arguments."""
import numpy as np

import statistic_cases
from statistic_oracle import ADD1, COUNT, COV, FIRST, MIN_MAX, MOMENTS_01, MOMENTS_012


def _case(binby, weights, op, sizes=(), minima=(), maxima=(), edges=False, selections=(None,)):
    return dict(binby=list(binby), weights=list(weights), selections=list(selections), op=op, sizes=list(sizes), minima=list(minima),
                maxima=list(maxima), edges=edges)


def _product_quirk_rows():
    """float32 values whose bin at size 777 differs between the float32 product (exactly two dimensions) and the double product"""
    rng = np.random.default_rng(7)
    s = rng.random(2_000_000).astype(np.float32)
    f32 = (s * np.float32(777)).astype(np.int64)
    f64 = (s.astype(np.float64) * 777).astype(np.int64)
    return s[f32 != f64][:16]


def cases():
    out = {}
    q = _product_quirk_rows()
    assert len(q) >= 4
    # the 2-D float32 product against the same rows binned in 1-D and 3-D (double product)
    out["kat_product_2d_f32"] = _case([q, q], [], ADD1, [777, 777], [0, 0], [1, 1])
    out["kat_product_1d_f32"] = _case([q], [], ADD1, [777], [0], [1])
    out["kat_product_3d_f32"] = _case([q, q, q], [], ADD1, [777, 5, 5], [0, 0, 0], [1, 1, 1])
    # every edge cell: NaN -> 0, below -> 1, at / above max -> size-1, at min -> 2
    e = np.array([np.nan, -1.0, 0.0, 0.25, 0.5, 0.999, 1.0, 2.0, np.inf, -np.inf], np.float64)
    out["kat_edges_f64"] = _case([e], [e], MOMENTS_012, [4 + 3], [0], [1], edges=True)
    out["kat_edges_f32"] = _case([e.astype(np.float32)], [e.astype(np.float32)], COUNT, [4 + 3], [0], [1], edges=True)
    # a NaN sum (inf - inf) that the MOMENTS reduce (nansum) turns into 0, and a NaN COV product that np.sum keeps
    inf = np.array([np.inf, -np.inf, 1.0], np.float64)
    out["kat_nan_sum_moments"] = _case([], [inf], MOMENTS_01)
    out["kat_nan_product_cov"] = _case([], [inf, np.array([1.0, 1.0, 2.0])], COV)
    # int32 / uint64 values rounded to float32 before binning and accumulation; int64 to float64
    i32 = np.array([16777217, -16777219, 2147483647, 3], np.int32)
    u64 = np.array([2**64 - 1, 2**53 + 1, 2**24 + 1, 5], np.uint64)
    i64 = np.array([2**53 + 1, -(2**62) - 1, 7, 0], np.int64)
    out["kat_round_int32_f32"] = _case([], [i32], MIN_MAX)
    out["kat_round_uint64_f32"] = _case([], [u64], MOMENTS_012)
    out["kat_round_int64_f64"] = _case([], [i64], MOMENTS_01)
    out["kat_round_int32_binby"] = _case([i32], [i32], MOMENTS_01, [4], [-2**31], [2**31])
    # FIRST: ties keep the earliest row, NaN and +inf orders never win, -0.0 ties +0.0
    v = np.array([10, 11, 12, 13, 14, 15, 16, 17], np.float64)
    o = np.array([3.0, 1.0, 1.0, np.nan, np.inf, -np.inf, 0.0, -0.0])
    out["kat_first_ties"] = _case([], [v[:5], o[:5]], FIRST)
    out["kat_first_neginf"] = _case([], [v, o], FIRST)
    out["kat_first_zeros"] = _case([], [v[6:], o[6:]], FIRST)
    out["kat_first_nan_inf_only"] = _case([], [v[3:5], o[3:5]], FIRST)
    # signed zeros where the reference's first-arrival rule and the device's -0 < +0 rule agree
    z = np.array([-0.0, 0.0, 0.0], np.float64)
    out["kat_signed_zeros_min"] = _case([], [z], MIN_MAX)
    out["kat_signed_zeros_sum"] = _case([], [np.array([-0.0, -0.0])], MOMENTS_012)
    rng = np.random.default_rng(4242)
    for k in range(12):
        out["random_%02d" % k] = statistic_cases.random_case(rng, n=500)
    return out
