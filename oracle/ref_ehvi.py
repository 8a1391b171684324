"""ctypes front-end of oracle/_ref/libref_ehvi.so: the reference's OWN ehvi2d, experimental::acqui::Ehvi over two of its GPs, and
pareto::pareto_set (oracle/ref_shim/ehvi_driver.cpp, built by oracle/ref_shim/Makefile).  TEST INFRASTRUCTURE ONLY; built only
where the reference's sources are present (oracle/ref.py: REF_SRC) — elsewhere the tests rely on tests/golden/ehvi/."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .ref import RefLibrary


def _declare(lib):
    vp, lg, i, d = C.c_void_p, C.c_long, C.c_int, C.c_double
    lib.ref_ehvi2d.argtypes = [lg, vp, vp, lg, vp, vp, vp]
    lib.ref_pareto_set.argtypes = [lg, i, vp, vp, vp]
    lib.ref_gp_ehvi.argtypes = [lg, i, vp, vp, d, vp, lg, vp, vp, vp, vp, vp, vp]
    for f in (lib.ref_ehvi2d, lib.ref_pareto_set, lib.ref_gp_ehvi):
        f.restype = i


_LIB = RefLibrary("libref_ehvi.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def _c(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a.reshape(shape) if shape is not None else a


def ehvi2d(front, r, mu, s) -> np.ndarray:
    """ehvi2d(front, r, mu_q, s_q) for M candidates: front k x 2, mu and s M x 2."""
    F, R, MU, S = _c(front, (-1, 2)), _c(r).reshape(-1)[:2].copy(), _c(mu, (-1, 2)), _c(s, (-1, 2))
    out = np.empty(MU.shape[0])
    assert load().ref_ehvi2d(F.shape[0], F.ctypes.data if F.size else None, R.ctypes.data, MU.shape[0], MU.ctypes.data,
                             S.ctypes.data, out.ctypes.data) == 0
    return out


def pareto_set(objs) -> np.ndarray:
    """pareto::pareto_set<1>: kept indices of the rows of objs (n x K) in the reference's order (ties unordered)."""
    O = _c(objs)
    idx = np.empty(O.shape[0], dtype=np.int64)
    nf = C.c_long()
    assert load().ref_pareto_set(O.shape[0], O.shape[1], O.ctypes.data, idx.ctypes.data, C.addressof(nf)) == 0
    return idx[: nf.value]


def gp_ehvi(X, Y, Xq, r=(-11.0, -11.0), noise=0.01) -> dict:
    """One Matern-5/2 / mean::Data GP per objective on (X, Y[:, j]) with default hyper-parameters, the Pareto set of Y and the
    reference's acqui::Ehvi at every candidate.  Returns ehvi, mu (M x 2), s (M x 2: sigma() = sigma^2 + noise) and front."""
    X, Y, Xq, R = _c(X), _c(Y, (-1, 2)), _c(Xq), _c(r).reshape(-1)[:2].copy()
    N, D = X.shape
    M = Xq.shape[0]
    out = {"ehvi": np.empty(M), "mu": np.empty((M, 2)), "s": np.empty((M, 2)), "front": np.empty((N, 2))}
    nf = C.c_long()
    assert load().ref_gp_ehvi(N, D, X.ctypes.data, Y.ctypes.data, float(noise), R.ctypes.data, M, Xq.ctypes.data,
                              *[out[k].ctypes.data for k in ("ehvi", "mu", "s", "front")], C.addressof(nf)) == 0
    out["front"] = out["front"][: nf.value].copy()
    return out
