"""Frame.join at key edges against the join restatement (join_oracle.join with bit-pattern keys): the sentinel key (the one whose
canonical pattern is the device table's empty marker), integer limits, uint64 >= 2^63, +-inf, subnormals, NaN payloads, NaT and the
int64 extremes of datetimes; left keys on the host, page-locked and on the device; executor splits that put the sentinel, NaN and null
rows into different chunks and threads; right lengths around the lookup's int8 / int16 / int32 boundaries; and left / right keys of
different dtypes."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import join_cases  # noqa: E402
import join_oracle as J  # noqa: E402
import set_cases as S  # noqa: E402
from test_gpu_index_hash import vector_duplicates  # noqa: E402
from test_gpu_join import DTYPES, same, to_frame, values  # noqa: E402

pytestmark = pytest.mark.gpu

PLACES = ["host", "pinned", "device"]
SPLITS = [(1, None), (8, 256), (3, 1000)]
N_LEFT = 3000


def _int64_like(dtype):
    return np.dtype(dtype).kind == "M"


def edge_keys(dtype):
    """every edge value and NaN payload of a key dtype (datetimes: the int64 edges as ticks, NaT = INT64_MIN among them)"""
    if _int64_like(dtype):
        return S.edge_values("int64").view(dtype)
    return np.concatenate([S.edge_values(dtype), S.nan_values(dtype)]).astype(dtype)


def sentinel(dtype):
    """the sentinel key of a dtype, or its largest value where it has none"""
    base = "int64" if _int64_like(dtype) else dtype
    s = S.sentinel(base)
    s = S.edge_values(base)[-1] if s is None else s
    return np.array([s], base).view(dtype)[0]


def distinct(dtype, n=400):
    if _int64_like(dtype):
        return dict((c[0], c[1]) for c in S.columns("int64", n=n))["distinct"].view(dtype)
    return dict((c[0], c[1]) for c in S.columns(dtype, n=n))["distinct"]


def right_side(dtype, dup, rng):
    """right keys: every edge value once (more than once with `dup`), the sentinel at its start, middle and end when duplicated, two
    NaN payloads and two masked rows in different chunks"""
    keys = distinct(dtype)
    if dup:
        keys = np.concatenate([keys, keys[: len(keys) // 4], [sentinel(dtype)] * 2]).astype(keys.dtype)
    rng.shuffle(keys)
    n = len(keys)
    s = sentinel(dtype)
    if dup:
        keys[[min(5, n - 2), n // 2, n - 1]] = s
    else:
        keys[np.flatnonzero(keys.view(f"u{keys.itemsize}") == np.array([s]).view(f"u{keys.itemsize}")[0])] = keys[n // 2]
        keys[n // 2] = s
    nans = S.nan_values(dtype) if not _int64_like(dtype) else np.zeros(0)
    mask = np.zeros(n, bool)
    if len(nans) and n > 10:
        keys[[n // 3, 2 * n // 3]] = nans[[1, 4]]
    if n > 10:
        mask[[n // 4, 3 * n // 4]] = True
    if not dup:  # no duplicate bit pattern (-0.0 and 0.0 are two keys)
        kept = keys[~mask & ~_isnan(keys)]
        assert len(np.unique(kept.view(f"u{kept.itemsize}"))) == len(kept)
    return {"k": np.ma.array(keys, mask=mask), "w": np.arange(n) * 0.5 + 0.25, "rx": np.arange(n, dtype=np.int64)}


def _isnan(k):
    return np.isnan(k) if k.dtype.kind == "f" else np.zeros(len(k), bool)


def left_side(dtype, right_keys, masked, rng):
    """left keys: the edge values, NaN payloads and never-inserted keys, then right keys; the sentinel at rows 0 / 1000 / 2999, NaN at
    rows 300 / 1700 and (when `masked`) nulls at rows 600 / 2600: different chunks at every split"""
    data = np.ma.getdata(right_keys)
    base = "int64" if _int64_like(dtype) else dtype
    q = S.queries(base).view(dtype) if _int64_like(dtype) else S.queries(dtype)
    keys = np.concatenate([q, data[rng.integers(0, len(data), N_LEFT - len(q))]]).astype(data.dtype)
    rng.shuffle(keys)
    keys[[0, 1000, N_LEFT - 1]] = sentinel(dtype)
    nans = S.nan_values(dtype) if not _int64_like(dtype) else np.zeros(0)
    if len(nans):
        keys[[300, 1700]] = nans[[0, 5]]
    cols = {"k": keys, "v": np.arange(N_LEFT) * 1.0}
    if masked:
        mask = np.zeros(N_LEFT, bool)
        mask[[600, 2600]] = True
        cols["k"] = np.ma.array(keys, mask=mask)
    return cols


def joined(left, right, rfilter, place, split, **kwargs):
    frames = [to_frame((left, None), place, *split), to_frame((right, rfilter), "host" if place == "device" else place, *split)]
    try:
        got = frames[0].join(frames[1], **kwargs)
        return {name: values(got, name, filtered=False) for name in got.columns}
    finally:
        for f in frames:
            if f._pinned is not None:
                f._pinned.release()


def oracle(left, right, rfilter, **kwargs):
    return J.join(J.OFrame(left), J.OFrame(right, join_cases.filter_mask(right, rfilter)), bits=True, **kwargs)


def check(got, want, what):
    assert set(got) == set(want.columns), what
    for name in want.columns:
        assert same(got[name], want.values(name, False)), (what, name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("how", ["left", "inner", "right"])
def test_edge_keys(dtype, how):
    rng = np.random.default_rng([DTYPES.index(dtype), ["left", "inner", "right"].index(how)])
    for dup, allow in ((False, False), (False, True), (True, True)):
        allow = allow or how == "right"  # a right join indexes the left side, whose keys repeat
        right = right_side(dtype, dup, rng)
        for place in PLACES:
            left = left_side(dtype, right["k"], place != "device", rng)
            for split, rfilter in zip(SPLITS, (None, "rx > 3", None) if how != "right" else (None,) * 3):
                kwargs = dict(on="k", how=how, rsuffix="_r", allow_duplication=allow)
                what = (dtype, how, dup, allow, place, split, rfilter)
                check(joined(left, right, rfilter, place, split, **kwargs), oracle(left, right, rfilter, **kwargs), what)
        if dup and how != "right":
            with pytest.raises(ValueError, match="duplication"):
                joined(left, right, None, "host", SPLITS[1], on="k", how=how, rsuffix="_r")


@pytest.mark.parametrize("masked", [False, True])
def test_datetime_nat_and_extremes(masked):
    """NaT is INT64_MIN of the int64 index (test_nat_is_an_ordinary_int64_key pins the compiled index_hash_int64 on this): a left NaT
    finds the right's NaT row, and the int64 extremes find theirs"""
    ticks = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, np.iinfo(np.int64).min + 1, -1, 0, 86_400 * 10 ** 9])
    right = {"k": ticks.view("M8[ns]"), "w": np.arange(len(ticks)) * 10}
    lt = np.concatenate([ticks[::-1], [5, ticks[0]]])
    mask = np.zeros(len(lt), bool)
    if masked:
        mask[[1, 6]] = True
        right["k"] = np.ma.array(right["k"], mask=np.eye(1, len(ticks), 2, dtype=bool)[0])
    left = {"k": np.ma.array(lt.view("M8[ns]"), mask=mask), "v": np.arange(len(lt))}
    for split in SPLITS:
        got = joined(left, right, None, "host", split, on="k", rsuffix="_r")
        check(got, oracle(left, right, None, on="k", rsuffix="_r"), split)
        want = [50, 40, 30, 20, 10, 0, None, 0]
        if masked:  # the masked left rows 1 and 6 find the right's null row 2, whose key MIN + 1 the left's row 3 then misses
            want = [50, 20, 30, None, 10, 0, 20, 0]
        assert got["w"] == want, (split, got["w"])


@pytest.mark.parametrize("n_right", [126, 127, 128, 32766, 32767, 32768, 65536])
def test_lookup_width_boundaries(n_right):
    """required_dtype_for_max(len(right)) switches the lookup int8 -> int16 -> int32 here; the lookup starts as iinfo.max, and with
    duplicates it is widened to int64 and extended"""
    rng = np.random.default_rng(n_right)
    for missing in (False, True):
        for dup in (False, True):
            rk = rng.permutation(n_right).astype(np.int64) * 3 - 7
            if dup:
                rk[-5:] = rk[:5]
            right = {"k": rk, "w": np.ma.array(np.arange(n_right) * 0.5, mask=np.arange(n_right) % 97 == 3), "c": (np.arange(n_right) % 251).astype(np.int16)}
            pick = rk[rng.integers(0, n_right, 4000)]
            if missing:
                pick[::7] = 3 * n_right + 1
            pick[[0, -1]] = [rk[0], rk[-1]]
            left = {"k": pick, "v": np.arange(len(pick))}
            want = oracle(left, right, None, on="k", rsuffix="_r", allow_duplication=True)
            for place, split in (("host", SPLITS[2]), ("device", SPLITS[1])):
                got = joined(left, right, None, place, split, on="k", rsuffix="_r", allow_duplication=True)
                check(got, want, (n_right, missing, dup, place))
                assert len(got["v"]) == len(pick) + (np.count_nonzero(np.isin(pick, rk[:5])) if dup else 0)


MATRIX = DTYPES


def _matrix_sides(ldtype, rdtype):
    rk = edge_keys(rdtype)
    lk = edge_keys(ldtype)
    lbase = lk.view(np.int64) if _int64_like(ldtype) else lk
    with np.errstate(invalid="ignore", over="ignore"):
        cast = lbase.astype("int64" if _int64_like(rdtype) else rdtype)
    rk = np.concatenate([rk, cast.view(rk.dtype) if _int64_like(rdtype) else cast]).astype(rk.dtype)
    right = {"k": rk, "w": np.arange(len(rk)) * 1.0}
    left = {"k": np.concatenate([lk, lk[::-1]]), "v": np.arange(2 * len(lk))}
    return left, right


@pytest.mark.parametrize("rdtype", MATRIX)
def test_mixed_key_dtypes(rdtype):
    """a left key of another dtype than the right's is cast by value where numpy calls the cast safe, and refused with a TypeError
    elsewhere; host, page-locked and device left keys give the same answer or the same error"""
    for ldtype in MATRIX:
        left, right = _matrix_sides(ldtype, rdtype)
        outcomes = []
        for place in PLACES:
            try:
                outcomes.append(joined(left, right, None, place, SPLITS[1], on="k", rsuffix="_r", allow_duplication=True))
            except TypeError as e:
                outcomes.append(("TypeError", "incompatible key dtype" in str(e)))
        what = (ldtype, rdtype)
        lb = np.dtype("int64") if _int64_like(ldtype) else np.dtype(ldtype)
        rb = np.dtype("int64") if _int64_like(rdtype) else np.dtype(rdtype)
        if np.can_cast(lb, rb, "safe"):
            want = oracle(left, right, None, on="k", rsuffix="_r", allow_duplication=True)
            for got in outcomes:
                assert not isinstance(got, tuple), (what, got)
                check(got, want, what)
        else:
            assert outcomes == [("TypeError", True)] * 3, (what, outcomes)


@pytest.mark.parametrize("dtype", ["uint64", "int32"])
def test_heavy_duplicates_of_the_sentinel(dtype):
    import torch
    rng = np.random.default_rng(3)
    s = S.sentinel(dtype)
    rk = rng.integers(0, 50_000, 2_000_000).astype(dtype)
    rk[rng.choice(len(rk), 300_000, replace=False)] = s
    lk = np.concatenate([rng.integers(0, 60_000, 3000).astype(dtype), np.full(3, s, dtype)])
    from vaex_b200 import superutils
    h = getattr(superutils, "index_hash_" + dtype)(3)
    for a in range(0, len(rk), 700_000):
        h.update(torch.from_numpy(rk[a:a + 700_000]).cuda(), a)
    left, right = h.map_index_duplicates(torch.from_numpy(lk).cuda(), 0, device=True)
    wl, wr = vector_duplicates(rk, lk, 0)
    assert np.array_equal(left.cpu().numpy(), wl) and np.array_equal(right.cpu().numpy(), wr)
    assert np.count_nonzero(lk == s) == 3
    first = np.flatnonzero(rk == s)[0]
    assert h.map_index(np.array([s], dtype)).tolist() == [first]
    # the whole join: every left sentinel row repeated for each of the right's sentinel rows, against an argsort join
    got = joined({"k": lk}, {"k": rk, "w": np.arange(len(rk), dtype=np.int64)}, None, "device", SPLITS[1], on="k", allow_duplication=True)
    lrows, rrows = J.numpy_join(lk, rk)
    assert np.array_equal(np.asarray(got["k"], dtype), lk[lrows])
    assert [None if r < 0 else r for r in rrows.tolist()] == got["w"]
