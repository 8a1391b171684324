"""Generates tests/golden/ehvi/*.npz: the REFERENCE'S OWN experimental::acqui::Ehvi over two of its GPs (oracle/_ref/libref_ehvi.so,
entry ref_gp_ehvi) and its raw ehvi2d (entry ref_ehvi2d) on seeded inputs, stored together with those inputs.  Models:
Matern-5/2 / mean::Data, P = 1, default hyper-parameters; reference point (-11, -11) as bayes_opt_ehvi's defaults.  Needs a built
oracle/_ref/libref_ehvi.so (oracle/ref_shim/Makefile: libref_ehvi.so):
    python tests/golden/make_golden_ehvi.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ehvi as E  # noqa: E402
from oracle import ref_ehvi  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ehvi")
R = np.array([-11.0, -11.0])
M = 500


def gp_case(name, X, Y, Xq, noise=0.01):
    r = ref_ehvi.gp_ehvi(X, Y, Xq, R, noise)
    np.savez_compressed(os.path.join(OUT, name), X=X, Y=Y, Xq=Xq, r=R, noise=noise, **r)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    rng = np.random.default_rng(2024)
    for N in (60, 300):
        X = rng.random((N, 2))
        gp_case(f"mop2_n{N}", X, E.mop2(X), rng.random((M, 2)))
        X = rng.random((N, 6))
        gp_case(f"zdt2_n{N}_d6", X, E.zdt2(X), rng.random((M, 6)))
    X = rng.random((40, 3))  # equal objectives: the front is the best point
    y = -((X - 0.5) ** 2).sum(axis=1)
    gp_case("front_k1", X, np.stack([y, y], axis=1), rng.random((M, 3)))
    X = rng.random((50, 2))
    X = np.concatenate([X, X[:12]])  # duplicated observations: the duplicates of front points stay in the front
    gp_case("duplicates", X, E.mop2(X), rng.random((M, 2)))
    X = rng.random((60, 2))  # candidates on the samples: sigma^2 + noise is small there
    gp_case("on_samples", X, E.mop2(X), X.copy(), noise=1e-6)
    # models without samples score with their prior: mu = 0 (mean::Data of nothing), s = sigma_f^2 + noise = 1.01
    front = E.mop2(rng.random((80, 2)))
    front = front[E.pareto_set(front)]
    mu, s = np.zeros((M, 2)), np.full((M, 2), 1.01)
    np.savez_compressed(os.path.join(OUT, "prior"), front=front, r=R, Xq=rng.random((M, 2)), mu=mu, s=s,
                        ehvi=ref_ehvi.ehvi2d(front, R, mu, s))
    # a raw front of 2000 points (mutually non-dominated) for ehvi2d alone
    k = 2000
    f0 = np.sort(rng.uniform(-10.0, 0.0, k))
    front = np.stack([f0, np.sort(rng.uniform(-10.0, 0.0, k))[::-1]], axis=1)[rng.permutation(k)]
    mu = rng.uniform(-11.0, 1.0, (16, 2))
    s = rng.uniform(0.05, 3.0, (16, 2))
    np.savez_compressed(os.path.join(OUT, "raw_k2000"), front=front, r=R, mu=mu, s=s, ehvi=ref_ehvi.ehvi2d(front, R, mu, s))
    print("wrote", OUT)
