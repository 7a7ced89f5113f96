"""Write tests/golden/lasso_golden.npz: for every case of lasso_oracle.corpus() the polygon, the rows and the mask of the compiled,
unmodified vaexfast.pnpoly (polygons of up to 1000 vertices), for the GPU tests (which cannot run the reference).  Run from the repository root after build()."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

import lasso_oracle  # noqa: E402
import ref_driver  # noqa: E402
from vaex_b200.selections import lasso_constants  # noqa: E402


def main():
    out = {}
    vf = ref_driver.vaexfast()
    for k, (name, xs, ys, bx, by) in enumerate(lasso_oracle.corpus()):
        if len(xs) > 1000:
            continue  # the 10^4-vertex lasso is checked against the restatement on the GPU; it would dominate the file
        vx, vy, meanx, meany, radius = lasso_constants(xs, ys)
        bx, by = np.ascontiguousarray(bx, np.float64), np.ascontiguousarray(by, np.float64)
        mask = np.zeros(len(bx), dtype=bool)
        vf.pnpoly(vx, vy, bx, by, mask, meanx, meany, radius)
        out[f"{k}_vx"], out[f"{k}_vy"], out[f"{k}_x"], out[f"{k}_y"], out[f"{k}_mask"] = vx, vy, bx, by, mask
        out[f"{k}_name"] = np.array(name)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "lasso_golden.npz"), **out)


if __name__ == "__main__":
    main()
