"""ctypes front-end of oracle/_ref/libref_eci.so: the reference's OWN experimental::acqui::ECI (oracle/ref_shim/eci_driver.cpp,
built by oracle/ref_shim/Makefile).  TEST INFRASTRUCTURE ONLY; built only where the reference's sources are present (oracle/ref.py:
REF_SRC) — elsewhere the tests rely on tests/golden/eci/."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .ref import RefLibrary


def _declare(lib):
    vp, lg, i, d = C.c_void_p, C.c_long, C.c_int, C.c_double
    lib.ref_gp_eci.argtypes = [i, lg, i, vp, vp, lg, vp, d, d, lg, vp] + [vp] * 6
    lib.ref_gp_eci.restype = i


_LIB = RefLibrary("libref_eci.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def eci(con_kernel_id: int, X, y, Yc, Xq, noise=0.01, jitter=0.0):
    """The reference's experimental::acqui::ECI over an SE-ARD / mean::Data objective GP on (X, y) and an Exp (3) or
    Matern-5/2 (1) / mean::Constant (0.25) constraint GP on the first len(Yc) samples (Yc: n x 2; n = 0: no constraint samples),
    default hyper-parameters.  Returns a dict with eci, mu, sigma2, mu_c (M x 2), sigma2_c and f_max."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    y = np.ascontiguousarray(y, dtype=np.float64).reshape(-1)
    Yc = np.ascontiguousarray(Yc, dtype=np.float64).reshape(-1, 2)
    Xq = np.ascontiguousarray(Xq, dtype=np.float64)
    N, D = X.shape
    M = Xq.shape[0]
    out = {"eci": np.empty(M), "mu": np.empty(M), "sigma2": np.empty(M), "mu_c": np.empty((M, 2)), "sigma2_c": np.empty(M)}
    f_max = C.c_double()
    rc = lib.ref_gp_eci(con_kernel_id, N, D, X.ctypes.data, y.ctypes.data, Yc.shape[0], Yc.ctypes.data if Yc.size else None,
                        float(noise), float(jitter), M, Xq.ctypes.data, *[out[k].ctypes.data for k in ("eci", "mu", "sigma2", "mu_c", "sigma2_c")],
                        C.addressof(f_max))
    assert rc == 0, rc
    out["f_max"] = f_max.value
    return out
