"""The numpy restatement of vaexfast.pnpoly (tests/lasso_oracle.py) against the compiled, unmodified reference over an edge corpus,
and the banded edge index of LassoPlan against the plain loop: a row that tests only its band's edges gets the same answer."""
import numpy as np
import pytest

import lasso_oracle as L
from vaex_b200.selections import LassoPlan, band_of, lasso_constants


def reference_pnpoly(ref, xseq, yseq, bx, by):
    vf = ref.vaexfast()
    vx, vy, meanx, meany, radius = lasso_constants(xseq, yseq)
    mask = np.zeros(len(bx), dtype=bool)
    vf.pnpoly(vx, vy, bx, by, mask, meanx, meany, radius)
    return mask


def banded(plan, tx, ty):
    """b200_lasso's banded loop, row by row on the host"""
    p = plan
    out = np.zeros(len(tx), bool)
    rsq = p.radius * p.radius
    with np.errstate(all="ignore"):
        for r, (x, y) in enumerate(zip(tx, ty)):
            dx, dy = x - p.meanx, y - p.meany
            if not dx * dx + dy * dy < rsq or not (p.lo <= y < p.hi):
                continue
            b = int(band_of(y, p.lo, p.scale, p.nbands))
            c = False
            for xi, yi, xj, yj in p.band_edges(b):
                if (yi > y) != (yj > y) and x < (xj - xi) * (y - yi) / (yj - yi) + xi:
                    c = not c
            out[r] = c
    return out


CORPUS = L.corpus()


@pytest.mark.parametrize("case", CORPUS, ids=[c[0] for c in CORPUS])
def test_restatement_equals_compiled_pnpoly(ref, case):
    _, xs, ys, bx, by = case
    want = reference_pnpoly(ref, xs, ys, np.ascontiguousarray(bx, np.float64), np.ascontiguousarray(by, np.float64))
    assert np.array_equal(L.lasso(xs, ys, bx, by), want)


@pytest.mark.parametrize("case", [c for c in CORPUS if len(c[1]) >= 3], ids=[c[0] for c in CORPUS if len(c[1]) >= 3])
def test_banded_index_equals_plain_loop(case):
    _, xs, ys, bx, by = case
    plan = LassoPlan(xs, ys, banded=True)
    n = min(len(bx), 1500)
    assert np.array_equal(banded(plan, bx[:n], by[:n]), L.lasso(xs, ys, bx[:n], by[:n]))


def test_band_boundary_rows():
    """rows exactly on every band boundary and one ulp either side"""
    xs, ys = L.polygon(200, seed=5)
    plan = LassoPlan(xs, ys, banded=True)
    assert plan.nbands > 1
    edges = plan.lo + np.arange(plan.nbands + 1) / plan.scale
    ty = np.concatenate([edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf)])
    ty = np.tile(ty, 3)
    tx = np.repeat([-0.3, 0.0, 0.4], len(ty) // 3)
    assert np.array_equal(banded(plan, tx, ty), L.lasso(xs, ys, tx, ty))


@pytest.mark.parametrize("dtype", ["float32", "int64", "uint64", ">f8", "masked"])
def test_row_dtypes(ref, dtype):
    """the reference converts a block with as_flat_float (a big-endian float64 is read through its byte order) and drops masked rows"""
    rng = np.random.default_rng(1)
    if dtype in ("int64", "uint64"):
        big = 2 ** 53 + rng.integers(0, 1000, 500)
        bx = big.astype(dtype)
        by = (big + rng.integers(-3, 3, 500)).astype(dtype)
        xs = [2.0 ** 53, 2.0 ** 53 + 1000, 2.0 ** 53 + 1000, 2.0 ** 53]
        ys = [2.0 ** 53 - 5, 2.0 ** 53 - 5, 2.0 ** 53 + 700, 2.0 ** 53 + 700]
    else:
        bx, by = rng.uniform(-2, 2, 500), rng.uniform(-2, 2, 500)
        xs, ys = L.polygon(12, seed=2)
        if dtype == "float32":
            bx, by = bx.astype("f4"), by.astype("f4")
        elif dtype == ">f8":
            bx, by = bx.astype(">f8"), by.astype(">f8")
    want_x, want_y = bx, by
    got = None
    if dtype == "masked":
        m = rng.random(500) < 0.2
        bx = np.ma.array(bx, mask=m)
        want = reference_pnpoly(ref, xs, ys, np.asarray(bx.data), by) & ~m
        got = L.lasso(xs, ys, bx, by)
    else:
        conv = [b if b.dtype.type == np.float64 else b.astype(np.float64) for b in (want_x, want_y)]  # vaex.utils.as_flat_float
        want = reference_pnpoly(ref, xs, ys, *conv)
        got = L.lasso(xs, ys, bx, by)
    assert want.any() and not want.all()
    assert np.array_equal(got, want)


def test_plan_choice_and_constants():
    xs, ys = L.polygon(63)
    assert not LassoPlan(xs, ys).banded
    xs, ys = L.polygon(64)
    p = LassoPlan(xs, ys)
    assert p.banded and p.band_start[0] == 0 and p.band_start[-1] == len(p.edges)
    x, y, meanx, meany, radius = lasso_constants(xs, ys)
    assert meanx == np.array(xs, np.float64).mean() and radius == np.sqrt((meanx - x) ** 2 + (meany - y) ** 2).max()
