"""The numpy restatement of the legacy statistics (tests/statistic_oracle.py) against the compiled, unmodified vaexfast, bit for bit,
and the committed golden vectors against the restatement."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import statistic_cases  # noqa: E402
import statistic_oracle as SO  # noqa: E402
from helpers import same_bits  # noqa: E402


@pytest.mark.parametrize("seed", range(60))
def test_oracle_matches_compiled_vaexfast(ref, seed):
    rng = np.random.default_rng(1000 + seed)
    case = statistic_cases.random_case(rng)
    chunk = int(rng.choice([None, 700]) or 0) or None
    want = SO.process(**case, chunk=chunk, impl="vaexfast")
    got = SO.process(**case, chunk=chunk, impl="oracle")
    assert got.shape == want.shape
    assert same_bits(got, want)


def test_golden_regenerates_byte_for_byte(tmp_path):
    out = tmp_path / "statistic_golden.npz"
    subprocess.check_call([sys.executable, os.path.join(HERE, "golden", "make_golden_statistic.py"), str(out)])
    assert out.read_bytes() == open(os.path.join(HERE, "golden", "statistic_golden.npz"), "rb").read()


def test_golden_against_oracle():
    from golden_statistic import cases
    g = np.load(os.path.join(HERE, "golden", "statistic_golden.npz"))
    for name, case in cases().items():
        assert same_bits(SO.process(**case), g[name]), name


def test_golden_cases_against_compiled_vaexfast(ref):
    from golden_statistic import cases
    for name, case in cases().items():
        assert same_bits(SO.process(**case, impl="vaexfast"), SO.process(**case)), name
