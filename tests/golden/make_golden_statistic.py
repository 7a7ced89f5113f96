"""Generate tests/golden/statistic_golden.npz: the legacy-statistic grids (before the op's reduce) of tests/golden_statistic.py's
cases, from the numpy restatement tests/statistic_oracle.py, which tests/test_statistic_oracle_cpu.py pins bit for bit against the
compiled vaexfast.

    python tests/golden/make_golden_statistic.py [out.npz]

The archive is written with fixed zip timestamps, so a rerun reproduces it byte for byte."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from golden_statistic import cases  # noqa: E402
from make_golden_edges import save  # noqa: E402
from statistic_oracle import process  # noqa: E402

if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "statistic_golden.npz")
    save(path, {name: process(**case) for name, case in cases().items()})
