"""Generates tests/golden/parego/*.npz: the REFERENCE'S OWN experimental::model::GPParego (oracle/_ref/libref_parego.so, entry
ref_parego, see oracle/ref_shim/parego_driver.cpp) over model::GP (Matern-5/2, mean::Data, default hyper-parameters, noise 0.01)
with replayed weight vectors, on seeded inputs, stored together with those inputs: the scalarised observations, mu and sigma^2
at the samples and at 200 query points, and UCB (alpha 0.5) and EI (jitter 0, f_max the largest mu at the samples) there.
Problems: MOP2 (D = 2) and ZDT2 (D = 6) of oracle/ehvi.py, with K = 3 adding -(f1 + f2) as a third, negative objective.
Needs the reference's sources (oracle/ref_parego.py builds the driver):
    python tests/golden/make_golden_parego.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from limbo_b200 import synth  # noqa: E402
from oracle import ehvi as OE, oracle as O, ref_parego  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "parego")
M = 200
# name: (problem, D, N, K, rho, n0: samples given to compute(), the rest added one by one with add_sample()): MOP2 (D = 2) and ZDT2
# (D = 6) at N = 60 and 300, K = 2 and 3, rho = 0.05 and 0, and one add_sample sequence
CASES = {f"{p}_n{N}_k{K}_rho{'0' if rho == 0 else '05'}": (p, D, N, K, rho, N)
         for p, D in (("mop2", 2), ("zdt2", 6)) for N in (60, 300) for K in (2, 3) for rho in (0.05, 0.0)}
CASES["mop2_add_n60_k2_rho05"] = ("mop2", 2, 60, 2, 0.05, 50)


def objectives(problem, X, K):
    F = OE.mop2(X) if problem == "mop2" else OE.zdt2(X)
    return np.concatenate([F, -(F[:, :1] + F[:, 1:2])], axis=1) if K == 3 else F


def inputs(problem, D, N, K, n0):
    X = synth.points(900 + N + D, N, D)
    Xq = synth.points(901 + N + D, M, D)
    draws = np.random.default_rng(N * 10 + D + K).random((1 + N - n0, K))
    return X, objectives(problem, X, K), Xq, draws


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for name, (problem, D, N, K, rho, n0) in CASES.items():
        X, F, Xq, draws = inputs(problem, D, N, K, n0)
        scal, mu, s2 = ref_parego.parego(X, F, draws, np.concatenate([X, Xq]), n0=n0, rho=rho)
        f_max = mu[:N].max()
        np.savez_compressed(os.path.join(OUT, name + ".npz"), X=X, F=F, Xq=Xq, draws=draws, n0=n0, rho=rho, scal=scal, mu_samples=mu[:N],
                            mu=mu[N:], sigma2=s2[N:], ucb=O.ucb(mu[N:], s2[N:], 0.5), ei=O.ei(mu[N:], s2[N:], f_max, 0.0), f_max=f_max)
        print(name, "ok")
