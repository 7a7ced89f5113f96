"""The sort restatement (sort_oracle.py) against pa.compute.sort_indices, the reference's argsort: arrow's rules for NaN, null,
±0.0, NaT, unsigned and bool keys, strings, byte order and stability, over an edge corpus of 1-4 keys in every direction."""
import itertools
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sort_oracle as S  # noqa: E402

pa = pytest.importorskip("pyarrow")

ALL = S.NUMERIC + S.TIMES + ["string"]


def check(keys):
    got, want = S.argsort(keys), S.arrow_argsort(keys)
    assert np.array_equal(got, want), (got.tolist(), want.tolist())


@pytest.mark.parametrize("dtype", ALL)
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("byteswap", [False, True])
@pytest.mark.parametrize("descending", [False, True])
def test_one_key(dtype, masked, byteswap, descending):
    rng = np.random.default_rng(zlib.crc32(repr((dtype, masked, byteswap, descending)).encode()))
    check([S.random_key(rng, dtype, 300, masked, byteswap, descending)])


@pytest.mark.parametrize("nkeys", [1, 2, 3, 4])
def test_every_direction_mix(nkeys):
    rng = np.random.default_rng(nkeys)
    for directions in itertools.product([False, True], repeat=nkeys):
        for trial in range(6):
            keys = [S.random_key(rng, rng.choice(ALL), 200, rng.random() < 0.5, rng.random() < 0.3, d) for d in directions]
            check(keys)


def test_random_tables():
    rng = np.random.default_rng(7)
    for trial in range(200):
        n = int(rng.integers(0, 60))
        check([S.random_key(rng, rng.choice(ALL), n, rng.random() < 0.5, rng.random() < 0.3, rng.random() < 0.5) for _ in range(rng.integers(1, 4))])


@pytest.mark.parametrize("descending", [False, True])
def test_the_rules(descending):
    """each of arrow's rules on its own, against sort_indices"""
    f = np.array([np.nan, 1.0, -0.0, 0.0, np.nan, -np.inf, np.inf, 0.0, -0.0], "f8")
    check([(f, None, descending)])                                                     # ±0 equal, NaN equal and last
    check([(f, np.arange(9) % 4 == 0, descending)])                                    # null after NaN
    check([(np.array([True, False, True, False]), None, descending)])                  # False < True
    check([(np.array([2 ** 63, 1, 2 ** 64 - 1, 0, 2 ** 63 - 1], "u8"), None, descending)])  # unsigned
    check([(np.array(["b", "", "ä", "a", "B", None], object), None, descending)])      # bytewise, null last
    check([(np.zeros(50, "i4"), None, descending)])                                    # all equal: row order
    nat = np.array([5, np.iinfo(np.int64).min, -3, 0], np.int64).view("M8[ns]")
    check([(nat, None, descending)])                                                   # NaT without a mask: null
    check([(nat, np.array([False, False, True, False]), descending)])                  # masked: an unmasked NaT is INT64_MIN


def test_nat_rule_is_arrows():
    """the two NaT conversions of the issue, pinned directly on arrow"""
    nat = np.array([np.iinfo(np.int64).min, 1], np.int64).view("M8[ns]")
    assert S.to_arrow(nat).null_count == 1
    assert S.to_arrow(nat, np.array([False, True])).to_pylist()[0] is not None


def test_empty():
    check([(np.zeros(0, "f4"), None, False)])
