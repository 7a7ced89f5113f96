"""Generate tests/golden/index_hash_edges_golden.npz: the sequential edge cases of tests/index_hash_edge_cases.py and what the compiled,
unmodified reference classes (oracle/_ref superutils, `make -C oracle ref`) return for them.

    python tests/golden/make_golden_index_hash_edges.py [out.npz]

Every dtype with each kind of case ("one_", "calls_", "merge_"), edge keys (the sentinel, integer limits, uint64 >= 2^63, +-inf,
subnormals, every NaN payload) with masks, several calls and merges in row order, every `out` width.  Each dtype takes two nmaps per
kind, rotated so that every kind meets every nmaps of set_cases.NMAPS over the dtypes; the whole dtype x nmaps product is compared
with the compiled classes directly (test_index_hash_edges_cpu.py), which needs no stored answers.  -0.0 is left out: whether the
compiled reference's equality merges it with 0.0 depends on where the two land in its table.  The layout, `run`, `flatten` and
`load` are make_golden_index_hash's; only inputs and outputs are stored."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import index_hash_edge_cases as E  # noqa: E402
import make_golden_index_hash as G  # noqa: E402

PATH = os.path.join(HERE, "index_hash_edges_golden.npz")


KINDS = ["one", "calls", "merge"]


def stored(dtype, nmaps, kind):
    """whether the golden file holds this case: nmaps positions d + 3k and d + 3k + 1 (mod 9) for dtype d and kind k"""
    d, k, m = E.DTYPES.index(dtype), KINDS.index(kind), E.NMAPS.index(nmaps)
    return (m - d - 3 * k) % len(E.NMAPS) in (0, 1)


def cases():
    return {name: c for name, c in E.all_sequential(zeros=False).items() if stored(c["dtype"], c["nmaps"], name.split("_")[0])}


def load(path=PATH):
    return G.load(path)


def main():
    from oracle import ref_driver
    from make_golden_edges import save
    su = ref_driver.modules()[1]
    path = sys.argv[1] if len(sys.argv) > 1 else PATH
    flat = {}
    all_cases = cases()
    for name, case in all_cases.items():
        flat.update(G.flatten(name, case, G.run(lambda dt: getattr(su, "index_hash_" + dt), case)))
    save(path, flat)
    print(f"wrote {path}: {len(all_cases)} cases")


if __name__ == "__main__":
    main()
