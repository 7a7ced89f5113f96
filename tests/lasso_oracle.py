"""vaexfast.pnpoly (src/vaexfast.cpp:1856-1874) restated in numpy, one vectorised step per edge in the reference's order, and the
lasso's host side (vaex/selections.py:178-191) around it; tests/test_lasso_oracle_cpu.py pins it to the compiled reference."""
import numpy as np


def pnpoly(vx, vy, tx, ty, meanx, meany, radius):
    """the mask pnpoly writes for float64 rows (tx, ty): inside by the crossing-number rule, and only where the squared distance to
    (meanx, meany) is below radius * radius (pow(d, 2) is d * d in the compiled reference)"""
    vx, vy = np.asarray(vx, np.float64), np.asarray(vy, np.float64)
    tx, ty = np.asarray(tx, np.float64), np.asarray(ty, np.float64)
    n = len(vx)
    c = np.zeros(len(tx), dtype=bool)
    with np.errstate(all="ignore"):
        for i in range(n):
            j = n - 1 if i == 0 else i - 1
            toggles = (vy[i] > ty) != (vy[j] > ty)
            cross = tx < (vx[j] - vx[i]) * (ty - vy[i]) / (vy[j] - vy[i]) + vx[i]
            c ^= toggles & cross
        dx, dy = tx - meanx, ty - meany
        inside = dx * dx + dy * dy < radius * radius
    return c & inside


def lasso(xseq, yseq, blockx, blocky):
    """SelectionLasso.evaluate's mask for blocks x, y without a previous selection: the rows with a masked x or y are not selected"""
    from vaex_b200.selections import lasso_constants
    vx, vy, meanx, meany, radius = lasso_constants(xseq, yseq)
    masks = [np.ma.getmaskarray(b) for b in (blockx, blocky) if np.ma.isMaskedArray(b)]
    bx, by = (np.asarray(b.data if np.ma.isMaskedArray(b) else b).astype(np.float64) for b in (blockx, blocky))
    out = pnpoly(vx, vy, bx, by, meanx, meany, radius)
    for m in masks:
        out &= ~m
    return out


def polygon(nvert, seed=0, kind="star"):
    """a closed lasso of nvert vertices around (0, 0): a star (radius varying per vertex), clockwise with kind="cw\""""
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 2 * np.pi, nvert, endpoint=False)
    r = 1 + 0.5 * rng.random(nvert)
    x, y = r * np.cos(t), r * np.sin(t)
    return (x[::-1].copy(), y[::-1].copy()) if kind == "cw" else (x, y)


def corpus():
    """(name, xseq, yseq, blockx, blocky): the edge cases of the lasso, rows and polygons"""
    rng = np.random.default_rng(7)
    sq = ([0.0, 2.0, 2.0, 0.0], [0.0, 0.0, 2.0, 2.0])
    grid = np.array([-1, -0.5, 0, 0.5, 1, 1.5, 2, 2.5, 3], np.float64)
    gx, gy = np.meshgrid(grid, grid)
    gx, gy = gx.ravel(), gy.ravel()
    out = [("square, on vertices and edges", *sq, gx, gy)]
    # the vertex (1, 3) of this triangle lies exactly on the bounding circle: the mean is (1, 1), the radius its distance 2
    tri = ([0.0, 2.0, 1.0], [0.0, 0.0, 3.0])
    out.append(("triangle, the vertex on the bounding circle", *tri, np.array([2.0, 0.0, 1.0, 1.0, 1.0]), np.array([0.0, 0.0, 3.0, 1.0, 1e-12])))
    special = np.array([np.nan, np.inf, -np.inf, 0.5, 1.0, -0.0, 0.0, 5e-324, 1 - 2 ** -53])
    sx, sy = np.meshgrid(special, special)
    out.append(("NaN and infinite rows", *sq, sx.ravel(), sy.ravel()))
    out.append(("NaN vertex", [0.0, np.nan, 2.0, 0.0], [0.0, 0.0, 2.0, 2.0], gx, gy))
    out.append(("infinite vertex", [0.0, np.inf, 2.0, 0.0], [0.0, 0.0, 2.0, 2.0], gx, gy))
    out.append(("clockwise square", sq[0][::-1], sq[1][::-1], gx, gy))
    out.append(("bow-tie", [0.0, 2.0, 0.0, 2.0], [0.0, 2.0, 2.0, 0.0], gx, gy))
    out.append(("repeated closing vertex", [0.0, 2.0, 2.0, 0.0, 0.0], [0.0, 0.0, 2.0, 2.0, 0.0], gx, gy))
    out.append(("one vertex", [1.0], [1.0], gx, gy))
    out.append(("two vertices", [0.0, 2.0], [0.0, 2.0], gx, gy))
    rx, ry = rng.uniform(-2, 2, 4000), rng.uniform(-2, 2, 4000)
    for nv in (3, 63, 64, 65, 1000, 10000):
        px, py = polygon(nv, seed=nv)
        # rows on the polygon's own vertices and on its y values (band boundaries fall there and between)
        bx = np.concatenate([rx, px, px[:50] + 1e-9, rng.uniform(-2, 2, len(py))])
        by = np.concatenate([ry, py, py[:50], py])
        out.append((f"star of {nv} vertices", px, py, bx, by))
    px, py = polygon(500, seed=3, kind="cw")
    out.append(("clockwise star", px, py, rx, ry))
    return out
