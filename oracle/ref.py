"""ctypes front-end of oracle/_ref/libref_gp.so: the reference's OWN GP code
(the src/limbo headers of a resibots/limbo checkout) compiled against the Eigen/Boost
stand-in (oracle/ref_shim/).  TEST INFRASTRUCTURE ONLY; built only where the reference's
sources are present (LIMBO_REFERENCE_SRC, default: a `reference` checkout next to this
repository) — elsewhere the tests rely on tests/golden/."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("LIMBO_REFERENCE_SRC", os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference", "src"))
REF_SRC = os.path.join(REF_ROOT, "limbo")


class RefLibrary:
    """One library under oracle/_ref/, built by its oracle/ref_shim/Makefile target where the reference's sources are present
    (make leaves it alone when it is up to date), loaded once, with the C signatures that declare(lib) sets."""

    def __init__(self, name: str, declare):
        self.name, self.path, self._declare, self._lib = name, os.path.join(HERE, "_ref", name), declare, None

    def available(self) -> bool:
        return os.path.exists(self.path) or os.path.isdir(REF_SRC)

    def load(self):
        if self._lib is None:
            if os.path.isdir(REF_SRC):
                subprocess.run(["make", "-C", os.path.join(HERE, "ref_shim"), "CXX=g++", f"REF={REF_ROOT}", self.name], check=True,
                               capture_output=True)
            lib = C.CDLL(self.path)
            self._declare(lib)
            self._lib = lib
        return self._lib


def _declare(lib):
    vp, lg, i, d = C.c_void_p, C.c_long, C.c_int, C.c_double
    lib.ref_gp_run.argtypes = [i, i, lg, i, i, vp, vp, d, vp, i, lg, lg, vp, i] + [vp] * 10
    lib.ref_gp_run.restype = i
    lib.ref_gp_loo.argtypes = [i, i, lg, i, i, vp, vp, d, vp, i, vp, vp]
    lib.ref_gp_loo.restype = i
    lib.ref_gp_mean_grad.argtypes = [i, lg, i, i, vp, vp, d, vp, i, vp, i, vp, vp, vp]
    lib.ref_gp_mean_grad.restype = i


_LIB = RefLibrary("libref_gp.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def run(kernel_id: int, X, Y, noise=0.01, hp=None, Xq=None, n0=0, rprop_iters=0, optimize_noise=False, want_grad=True):
    """Returns a dict with K, L, alpha, mu (incl. mean::Data), sigma2, loglik, grad, ucb, ei, hp."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    N, D = X.shape
    P = Y.shape[1]
    Xq = np.zeros((0, D)) if Xq is None else np.ascontiguousarray(Xq, dtype=np.float64)
    M = Xq.shape[0]
    nh_own = D + 1 if kernel_id == 0 else (3 * D + 1 if kernel_id == 4 else 2)  # 4 = SE-ARD with k = 2 Lambda columns
    nh = nh_own + (1 if optimize_noise else 0)
    hpa = None if hp is None else np.ascontiguousarray(hp, dtype=np.float64)
    K = np.empty((N, N), order="F"); L = np.empty((N, N), order="F"); A = np.empty((N, P), order="F")
    mu = np.empty((M, P)); s2 = np.empty(M); ll = C.c_double(); g = np.empty(nh); ucb = np.empty(M); ei = np.empty(M)
    hp_out = np.empty(nh)
    p = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    rc = lib.ref_gp_run(kernel_id, int(optimize_noise), N, D, P, p(X), p(Y), float(noise), p(hpa), 0 if hpa is None else hpa.size,
                        n0, M, p(Xq), rprop_iters, p(K), p(L), p(A), p(mu), p(s2), C.addressof(ll), p(g) if want_grad else None,
                        p(ucb), p(ei), p(hp_out))
    assert rc == 0, rc
    return {"K": K, "L": L, "alpha": A, "mu": mu, "sigma2": s2, "loglik": ll.value, "grad": g if want_grad else None,
            "ucb": ucb, "ei": ei, "hp": hp_out}


def loo(kernel_id: int, X, Y, noise=0.01, hp=None, optimize_noise=False, want_grad=True):
    """The reference's compute_log_loo_cv / compute_kernel_grad_log_loo_cv (gp.hpp:339-399)."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    N, D = X.shape
    nh = (D + 1 if kernel_id == 0 else (3 * D + 1 if kernel_id == 4 else 2)) + (1 if optimize_noise else 0)
    hpa = None if hp is None else np.ascontiguousarray(hp, dtype=np.float64)
    v = C.c_double()
    g = np.empty(nh)
    rc = lib.ref_gp_loo(kernel_id, int(optimize_noise), N, D, Y.shape[1], X.ctypes.data, Y.ctypes.data, float(noise),
                        None if hpa is None else hpa.ctypes.data, 0 if hpa is None else hpa.size, C.addressof(v),
                        g.ctypes.data if want_grad else None)
    assert rc == 0, rc
    return v.value, (g if want_grad else None)


def mean_grad(kernel_id: int, X, Y, mean_hp, noise=0.01, hp=None):
    """The reference's compute_log_lik / compute_mean_grad_log_lik (gp.hpp:313-330) with
    mean::FunctionARD<Params, mean::Constant<Params>>; mean_hp = [tr (P x (P+1) row-major), constant]."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    Y = np.ascontiguousarray(Y, dtype=np.float64)
    if Y.ndim == 1:
        Y = Y[:, None]
    N, D = X.shape
    P = Y.shape[1]
    hpa = None if hp is None else np.ascontiguousarray(hp, dtype=np.float64)
    mh = np.ascontiguousarray(mean_hp, dtype=np.float64)
    ll = C.c_double()
    g = np.empty(mh.size)
    mu0 = np.empty(P)
    rc = lib.ref_gp_mean_grad(kernel_id, N, D, P, X.ctypes.data, Y.ctypes.data, float(noise), None if hpa is None else hpa.ctypes.data,
                              0 if hpa is None else hpa.size, mh.ctypes.data, mh.size, C.addressof(ll), g.ctypes.data, mu0.ctypes.data)
    assert rc == 0, rc
    return ll.value, g, mu0
