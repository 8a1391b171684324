"""Restatement of experimental::acqui::ECI (experimental/acqui/eci.hpp:76-130) per candidate, FirstElem aggregator, in the
reference's own order of fp64 operations (Python floats are IEEE doubles; math.exp / math.erfc / math.sqrt are the C library's,
which the reference calls too).  TEST INFRASTRUCTURE ONLY: the product package limbo_b200/ never imports this."""
from __future__ import annotations

import math

import numpy as np


def eci_one(mu0: float, sigma2: float, mu_c0: float, sigma2_c: float, f_max: float, jitter: float, obj_empty: bool = False,
            con_empty: bool = False) -> float:
    """ECI of one candidate from the objective's mu[0] / sigma^2 and the constraint model's mu_c[0] / sigma_c^2 (means included).
    obj_empty / con_empty: that model has no samples (ECI = 0, resp. Pf = 1)."""
    sigma = math.sqrt(sigma2)
    if sigma < 1e-10 or obj_empty:  # eci.hpp:86
        return 0.0
    X = mu0 - f_max - jitter  # eci.hpp:101-104
    Z = X / sigma
    phi = math.exp(-0.5 * math.pow(Z, 2.0)) / math.sqrt(2.0 * math.pi)
    Phi = 0.5 * math.erfc(-Z / math.sqrt(2))
    pf = 1.0  # eci.hpp:116-130
    sigma_c = math.sqrt(sigma2_c)
    if not (sigma_c < 1e-10 or con_empty):
        pf = 0.5 * math.erfc(-((mu_c0 - 1.0) / sigma_c) / math.sqrt(2))
    return pf * (X * Phi + sigma * phi)  # eci.hpp:106


def eci(mu0, sigma2, mu_c0, sigma2_c, f_max, jitter=0.0, obj_empty=False, con_empty=False) -> np.ndarray:
    """eci_one over arrays of candidates."""
    a = [np.asarray(x, dtype=np.float64).reshape(-1) for x in (mu0, sigma2, mu_c0, sigma2_c)]
    return np.array([eci_one(float(m), float(s), float(mc), float(sc), float(f_max), float(jitter), bool(obj_empty), bool(con_empty))
                     for m, s, mc, sc in zip(*a)])
