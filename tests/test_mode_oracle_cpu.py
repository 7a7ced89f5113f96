"""The numpy restatement of df.mode (tests/mode_oracle.py) against the committed golden vectors (the reference's own method over the
compiled vaexfast histograms), and against the compiled vaexfast itself where oracle/_ref exists."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import mode_oracle as MO  # noqa: E402
from helpers import same_bits  # noqa: E402

REFERENCE_VAEX = "/root/reference/packages/vaex-core/vaex"
have_reference = pytest.mark.skipif(not os.access(os.path.join(REFERENCE_VAEX, "dataframe.py"), os.R_OK),
                                    reason="the reference sources are not on this machine")


def golden_columns(columns, case):
    if case["filter"]:
        keep = np.asarray(columns[case["filter"]], bool)
        return {k: v[keep] for k, v in columns.items()}
    return columns


def kwargs_of(case):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_mode import from_json
    return from_json(case["kwargs"])


def test_golden_against_restatement():
    columns, cases = MO.load_golden()
    assert len(cases) >= 35
    assert sum(not c["reference"] for c in cases.values()) == 4  # the departures of DESIGN.md section 3
    for name, case in cases.items():
        cols = golden_columns(columns, case)
        kwargs = kwargs_of(case)
        if "error" in case:
            with pytest.raises(Exception) as info:
                with np.errstate(all="ignore"):
                    MO.mode(cols, **kwargs)
            assert type(info.value).__name__ == case["error"], name
            continue
        with np.errstate(all="ignore"):
            got = MO.mode(cols, **kwargs)
        assert got.shape == case["result"].shape and got.dtype == case["result"].dtype, name
        assert same_bits(got, case["result"]), name


def test_golden_known_answers():
    columns, cases = MO.load_golden()
    assert cases["empty_binby"]["error"] == "ValueError" and cases["mode_shape_1"]["error"] == "IndexError"
    assert cases["four_d_unequal"]["error"] == "ValueError"
    assert np.all(np.isnan(cases["defaults_nonfinite_limits"]["result"]))  # histogram2d counts nothing with an infinite limit
    assert cases["three_d_unequal"]["result"].shape == (5, 7)  # indexed [b2, b1]: b1 = z is binned with the last size
    t = cases["ties"]["result"]
    assert np.allclose(t, 0.15)  # 0.1 and 0.6 tie in every cell: the first maximum, the center of bin 1 of [0, 1) in 10
    # the masked rows hold 50.0 under their mask and are counted there, in bin (50 + 3) / 63 * 16 = 13 of the mode axis
    m = columns["m"]
    counts = MO.histogram([columns["z"], m], [(0, 1), (-3, 60)], (16, 6))
    assert counts[13].sum() == np.ma.getmaskarray(m).sum() > 0


def counts_of(columns, binby, expression, limits, shape):
    return MO.histogram([columns[e] for e in binby + [expression]], limits, shape)


def test_value_edges():
    below = np.nextafter(1.0, 0.0)
    v = np.array([-1.0, 1.0, below, np.nan, np.inf, -np.inf])
    z = np.full(len(v), 0.5)
    # 2-D: at min -> bin 0; at max, NaN and +-inf dropped; just below max: scaled = 2 * 0.5 = 1.0 is not < 1, dropped
    c2 = MO.histogram([z, v], [(0, 1), (-1, 1)], (64, 2))
    assert c2.sum() == 1 and c2[0, 1] == 1
    # 3-D: just below max rounds (v - min) up to max - min, so the bin is 64: the last bin here
    c3 = MO.histogram([z, z, v], [(0, 1), (0, 1), (-1, 1)], (64, 2, 2))
    assert c3.sum() == 2 and c3[0, 1, 1] == 1 and c3[63, 1, 1] == 1
    # limits [0, 1]: just below max is bin 63 without rounding up in either rule
    assert MO.histogram([z, v], [(0, 1), (0, 1)], (64, 2))[63, 1] == 1
    assert MO.histogram([z, z, v], [(0, 1), (0, 1), (0, 1)], (64, 2, 2))[63, 1, 1] == 1


def test_nonfinite_limits():
    z = np.linspace(0, 0.9, 10)
    assert MO.histogram([z, z], [(0, 1), (0, np.inf)], (4, 4)).sum() == 0  # 2-D: nothing at all
    assert MO.histogram([z, z, z], [(0, 1), (0, 1), (-np.inf, 1)], (4, 4, 4)).sum() == 0  # inf * 0 = NaN: every row dropped
    c = MO.histogram([z, z, z], [(0, 1), (0, 1), (0, np.inf)], (4, 4, 4))
    assert c.sum() == 10 and c[0].sum() == 10  # scale 4 / inf = 0: every row in bin 0


@pytest.fixture
def vaexfast(ref):
    return ref.vaexfast()


def test_histograms_match_vaexfast(vaexfast):
    """the restatement's grid equals the compiled histogram2d / histogram3d / histogramNd on seeded data: 2-, 3- and 4-D, unequal
    shapes, values at min, at max and just below max (limits where nothing rounds up), NaN, +-inf, masked values"""
    rng = np.random.default_rng(7)
    n = 5000
    below = np.nextafter(1.0, 0.0)
    for trial in range(12):
        D = 2 + trial % 3
        shape = (4,) * D if D == 4 else tuple(int(s) for s in rng.integers(1, 40, D))
        blocks = []
        for _ in range(D):
            a = rng.random(n) * 1.2 - 0.1
            a[rng.random(n) < 0.05] = np.nan
            a[rng.random(n) < 0.02] = rng.choice([0.0, 1.0, below, np.inf, -np.inf])
            blocks.append(a)
        masked = np.ma.array(blocks[0], mask=rng.random(n) < 0.3)
        blocks[0] = masked
        limits = [(0.0, 1.0)] * D
        data = np.zeros(shape)
        raw = [np.ascontiguousarray(np.ma.getdata(b)) for b in blocks]
        flat = [v for lim in limits for v in lim]
        if D == 2:
            vaexfast.histogram2d(raw[0], raw[1], None, data, *flat)
        elif D == 3:
            vaexfast.histogram3d(raw[0], raw[1], raw[2], None, data, *flat)
        else:
            vaexfast.histogramNd(raw, None, data, [0.0] * D, [1.0] * D)
        assert np.array_equal(MO.histogram(blocks, limits, shape), data), (D, shape)
    # non-finite limits in 2-D: both count nothing
    data = np.zeros((3, 3))
    vaexfast.histogram2d(raw[0], raw[1], None, data, 0.0, np.inf, 0.0, 1.0)
    assert data.sum() == 0 and MO.histogram(blocks[:2], [(0, np.inf), (0, 1)], (3, 3)).sum() == 0


@have_reference
def test_golden_regenerates_byte_for_byte(ref, tmp_path):
    out = tmp_path / "mode_golden.npz"
    subprocess.check_call([sys.executable, os.path.join(HERE, "golden", "make_golden_mode.py"), str(out), REFERENCE_VAEX],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert out.read_bytes() == open(MO.GOLDEN, "rb").read()
