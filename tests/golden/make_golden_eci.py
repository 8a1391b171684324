"""Generates tests/golden/eci/*.npz: the REFERENCE'S OWN experimental::acqui::ECI (oracle/_ref/libref_eci.so, entry ref_gp_eci,
see oracle/ref_shim/eci_driver.cpp) on seeded inputs, stored together with those inputs.  Objective: SE-ARD / mean::Data, P = 1;
constraint: Exp or Matern-5/2 / mean::Constant (constant 0.25), P = 2; default hyper-parameters; 500 candidates.  Needs a built
oracle/_ref/libref_eci.so (oracle/ref_shim/eci.mk):
    python tests/golden/make_golden_eci.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from limbo_b200 import synth  # noqa: E402
from oracle import ref_eci  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "eci")
NOISE = 0.01
M = 500
# name: (constraint kernel id (1 Matern-5/2, 3 Exp), N, D, constraint samples, jitter)
CASES = {
    "exp_n60_d3": (3, 60, 3, 60, 0.0),
    "matern52_n130_d4": (1, 130, 4, 130, 0.0),
    "con_empty_n60_d3": (3, 60, 3, 0, 0.0),
    "exp_jitter_n60_d3": (3, 60, 3, 60, 1e3),  # every value underflows to 0: the argmax is index 0
}


def inputs(N, D, Nc):
    X = synth.points(500 + N, N, D)
    y = synth.targets(X)
    Yc = np.stack([0.2 + 1.6 * X[:Nc, 0], 2.0 - 1.5 * X[:Nc, 1]], axis=1)  # first column around the threshold 1
    Xq = synth.points(501 + N, M, D)
    return X, y, Yc, Xq


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for name, (ck, N, D, Nc, jitter) in CASES.items():
        X, y, Yc, Xq = inputs(N, D, Nc)
        r = ref_eci.eci(ck, X, y, Yc, Xq, NOISE, jitter)
        np.savez_compressed(os.path.join(OUT, name), X=X, y=y, Yc=Yc, Xq=Xq, con_kernel=ck, noise=NOISE, jitter=jitter,
                            **{k: np.asarray(v) for k, v in r.items()})
    print("wrote", OUT)
