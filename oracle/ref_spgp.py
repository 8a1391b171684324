"""ctypes front-end of oracle/_ref/libref_spgp.so: the reference's OWN experimental::model::SPGP (oracle/ref_shim/spgp_driver.cpp,
built by oracle/ref_shim/Makefile).  TEST INFRASTRUCTURE ONLY; built only where the reference's sources are present
(oracle/ref.py: REF_SRC) — elsewhere the tests rely on tests/golden/spgp/."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .ref import RefLibrary


def _declare(lib):
    vp, lg, i = C.c_void_p, C.c_long, C.c_int
    lib.ref_spgp.argtypes = [lg, i, vp, vp, lg, vp, lg, vp] + [vp] * 7
    lib.ref_spgp.restype = i


_LIB = RefLibrary("libref_spgp.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def run(X, y, M: int, w, Xq):
    """The reference at a fixed w: _likelihood(w, true) -> (f, grad); _compute(false) -> L, Lm, bet; _predict(Xq) -> mu (mean(v)
    included: mean::Data, the observations' mean) and sigma^2."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X[:, None]
    N, D = X.shape
    y = np.ascontiguousarray(y, dtype=np.float64).reshape(-1)
    w = np.ascontiguousarray(w, dtype=np.float64)
    Xq = np.ascontiguousarray(Xq, dtype=np.float64).reshape(-1, D)
    nq = Xq.shape[0]
    f = C.c_double()
    grad = np.empty(w.size)
    mu, s2 = np.empty(nq), np.empty(nq)
    L, Lm, bet = np.empty((M, M), order="F"), np.empty((M, M), order="F"), np.empty(M)
    rc = lib.ref_spgp(N, D, X.ctypes.data, y.ctypes.data, M, w.ctypes.data, nq, Xq.ctypes.data, C.addressof(f), grad.ctypes.data,
                      mu.ctypes.data, s2.ctypes.data, L.ctypes.data, Lm.ctypes.data, bet.ctypes.data)
    assert rc == 0, rc
    return {"f": f.value, "grad": grad, "mu": mu, "s2": s2, "L": L, "Lm": Lm, "bet": bet}
