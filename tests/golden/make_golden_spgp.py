"""Generate tests/golden/spgp/*.npz from the reference's OWN experimental::model::SPGP (oracle/ref_spgp.py, built by
oracle/ref_shim/Makefile as libref_spgp.so against the Eigen stand-in).  Each file stores X, y, M, w, the jitter, the _likelihood
value f and gradient, the _compute(false) factors L, Lm and bet at w, and mu (mean(v) included) / sigma^2 of _predict on 500
candidates Xq.
w is the reference's starting vector for a seeded permutation, moved off the start so that no pseudo-input sits on a sample.
Run from the repository root: python tests/golden/make_golden_spgp.py"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from limbo_b200 import synth  # noqa: E402
from oracle import ref_spgp  # noqa: E402
from oracle import spgp as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "spgp")
JITTER = 1e-6  # Params::model_spgp::jitter() of the driver (the reference default)


def cases():
    rng = np.random.default_rng(20261016)
    X = rng.uniform(0.0, 6.0, (100, 1))
    yield "cos1d_n100", X, np.cos(X[:, 0]), rng.uniform(0.0, 6.0, (500, 1))
    for name, N, D in (("n40_d2", 40, 2), ("n41_d2_odd", 41, 2), ("n5_d2_m1", 5, 2), ("n300_d3", 300, 3)):
        X = rng.uniform(0.0, 1.0, (N, D))
        yield name, X, np.sin(3.0 * X).sum(axis=1) + 0.05 * rng.normal(size=N), rng.uniform(0.0, 1.0, (500, D))
    X = synth.points(2026, 2000, 6)
    yield "hartmann6_n2000", X, synth.targets(X), synth.points(2027, 500, 6)


def main():
    os.makedirs(OUT, exist_ok=True)
    for k, (name, X, y, Xq) in enumerate(cases()):
        N, D = X.shape
        M = O.n_pseudo(N)
        rng = np.random.default_rng(k)
        w = O.init_w(X, y - y.mean(), M, rng.permutation(N)) + rng.normal(0.0, 0.05, (M + 1) * D + 2)
        r = ref_spgp.run(X, y, M, w, Xq)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), X=X, y=y, M=np.int64(M), w=w, jitter=np.float64(JITTER), Xq=Xq, f=r["f"],
                            grad=r["grad"], L=r["L"], Lm=r["Lm"], bet=r["bet"], mu=r["mu"], s2=r["s2"])
        print(name, X.shape, M, r["f"])


if __name__ == "__main__":
    main()
