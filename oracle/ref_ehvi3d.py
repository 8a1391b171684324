"""ctypes front-end of oracle/_ref/libref_ehvi3d.so: the reference's OWN ehvi3d_sliceupdate, ehvi3d_5term, ehvi3d_8term and hvol3d
(oracle/ref_shim/ehvi3d_driver.cpp, built by oracle/ref_shim/Makefile).  TEST INFRASTRUCTURE ONLY; built only where the
reference's sources are present (oracle/ref.py: REF_SRC) — elsewhere the tests rely on tests/golden/ehvi3d/."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .ref import RefLibrary


def _declare(lib):
    vp, lg, i = C.c_void_p, C.c_long, C.c_int
    for f in (lib.ref_ehvi3d_sliceupdate, lib.ref_ehvi3d_5term, lib.ref_ehvi3d_8term):
        f.argtypes = [lg, vp, vp, lg, vp, vp, vp]
        f.restype = i
    lib.ref_hv3d.argtypes = [lg, vp, vp, vp]
    lib.ref_hv3d.restype = i
    lib.ref_gp_ehvi3d.argtypes = [lg, i, vp, vp, C.c_double, vp, lg, vp, vp, vp, vp, vp, vp]
    lib.ref_gp_ehvi3d.restype = i


_LIB = RefLibrary("libref_ehvi3d.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def _c(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a.reshape(shape) if shape is not None else a


def _scheme(name, front, r, mu, s) -> np.ndarray:
    F, R, MU, S = _c(front, (-1, 3)), _c(r).reshape(-1)[:3].copy(), _c(mu, (-1, 3)), _c(s, (-1, 3))
    out = np.empty(MU.shape[0])
    assert getattr(load(), name)(F.shape[0], F.ctypes.data if F.size else None, R.ctypes.data, MU.shape[0], MU.ctypes.data,
                                 S.ctypes.data, out.ctypes.data) == 0
    return out


def ehvi3d_sliceupdate(front, r, mu, s) -> np.ndarray:
    """ehvi3d_sliceupdate(front, r, mu_q, s_q) for M candidates: front k x 3 (passed in its row order), mu and s M x 3."""
    return _scheme("ref_ehvi3d_sliceupdate", front, r, mu, s)


def ehvi3d_5term(front, r, mu, s) -> np.ndarray:
    return _scheme("ref_ehvi3d_5term", front, r, mu, s)


def ehvi3d_8term(front, r, mu, s) -> np.ndarray:
    return _scheme("ref_ehvi3d_8term", front, r, mu, s)


def hv3d(front, r) -> float:
    """hvol3d: the volume the front dominates between r and +inf."""
    F, R = _c(front, (-1, 3)), _c(r).reshape(-1)[:3].copy()
    out = C.c_double()
    assert load().ref_hv3d(F.shape[0], F.ctypes.data if F.size else None, R.ctypes.data, C.addressof(out)) == 0
    return out.value


def gp_ehvi3d(X, Y, Xq, r=(-11.0, -11.0, -11.0), noise=0.01) -> dict:
    """One Matern-5/2 / mean::Data GP per objective on (X, Y[:, j]) with default hyper-parameters (no rows: prior models), the
    reference's Pareto set of Y and ehvi3d_sliceupdate at every candidate with each model's mu(v)(0) and sigma(v).  Returns ehvi,
    mu (M x 3), s (M x 3) and front."""
    Xq = _c(Xq)
    D = Xq.shape[1]
    X, Y, R = _c(X).reshape(-1, D), _c(Y, (-1, 3)), _c(r).reshape(-1)[:3].copy()
    N, M = X.shape[0], Xq.shape[0]
    out = {"ehvi": np.empty(M), "mu": np.empty((M, 3)), "s": np.empty((M, 3)), "front": np.empty((max(N, 1), 3))}
    nf = C.c_long()
    assert load().ref_gp_ehvi3d(N, D, X.ctypes.data if N else None, Y.ctypes.data if N else None, float(noise), R.ctypes.data, M,
                                Xq.ctypes.data, *[out[k].ctypes.data for k in ("ehvi", "mu", "s", "front")], C.addressof(nf)) == 0
    out["front"] = out["front"][: nf.value].copy()
    return out
