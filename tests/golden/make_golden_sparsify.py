"""Generate tests/golden/sparsify/*.npz from the reference's OWN model::SparsifiedGP::_sparsify (oracle/ref_sparse.py, built by
oracle/ref_shim/sparse.mk against the Eigen stand-in).  Each file stores X, max_points, the kept indices, the removal order and the
density of every removed point when it was chosen.  Run from the repository root: python tests/golden/make_golden_sparsify.py"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_sparse  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sparsify")


def cases():
    rng = np.random.default_rng(20261015)
    # test_gp.cpp:760-880: M = 100 one-dimensional samples, max_points M / 3 and M / 2
    yield "gp1d_m100_max33", rng.uniform(0.0, 10.0, (100, 1)), 33
    yield "gp1d_m100_max50", rng.uniform(-2.0, 2.0, (100, 1)), 50
    yield "n500_d3_max200", rng.uniform(-1.0, 1.0, (500, 3)), 200  # the default max_points
    yield "n2000_d6_max1000", rng.uniform(0.0, 1.0, (2000, 6)), 1000
    # integer lattice: many exactly equal densities, so the lowest-index rule decides most removals
    g = np.stack(np.meshgrid(np.arange(16.0), np.arange(16.0), indexing="ij"), -1).reshape(-1, 2)
    yield "lattice16x16_max64", g, 64
    yield "n300_d4_max299", rng.normal(size=(300, 4)), 299  # one removal: the add_sample steady state
    yield "n50_d2_max200", rng.uniform(0.0, 1.0, (50, 2)), 200  # N <= max_points: nothing removed


def main():
    os.makedirs(OUT, exist_ok=True)
    for name, X, m in cases():
        kept, removed, score = ref_sparse.sparsify(X, m)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), X=X, max_points=np.int64(m), kept=kept, removed=removed,
                            removed_score=score)
        print(name, X.shape, m, len(kept), len(removed))


if __name__ == "__main__":
    main()
