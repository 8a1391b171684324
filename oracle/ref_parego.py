"""ctypes front-end of oracle/_ref/libref_parego.so: the reference's OWN experimental::model::GPParego with replayed weight
vectors (oracle/ref_shim/parego_driver.cpp and oracle/ref_shim/parego_shim).  TEST INFRASTRUCTURE ONLY; built by build() where
the reference's sources are present (oracle/ref.py: REF_SRC) — elsewhere the tests rely on tests/golden/parego/."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .ref import REF_ROOT, REF_SRC

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM = os.path.join(HERE, "ref_shim")
LIB_PATH = os.path.join(HERE, "_ref", "libref_parego.so")
_lib = None


def build() -> str:
    """compiles the driver with oracle/ref_shim/Makefile's library flags, the replaying shim first on the include path"""
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    subprocess.run(["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-fno-fast-math", "-ffp-contract=off", "-DNDEBUG", "-w",
                    "-I", os.path.join(SHIM, "parego_shim"), "-I", SHIM, "-I", REF_ROOT, "-shared", "-o", LIB_PATH,
                    os.path.join(SHIM, "parego_driver.cpp"), "-pthread"], check=True, capture_output=True)
    return LIB_PATH


def available() -> bool:
    return os.path.exists(LIB_PATH) or os.path.isdir(REF_SRC)


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        vp, lg, i, d = C.c_void_p, C.c_long, C.c_int, C.c_double
        lib.ref_parego.argtypes = [lg, lg, i, i, vp, vp, vp, d, d, lg, vp, vp, vp, vp]
        lib.ref_parego.restype = i
        _lib = lib
    return _lib


def parego(X, F, draws, Xq, n0=None, rho=0.05, noise=0.01):
    """The reference's GPParego (Matern-5/2, mean::Data, default hyper-parameters) after compute() on the first n0 samples (all by
    default) and add_sample() for each of the others, draws[c] (K raw weights) feeding call c.  Returns (scalarised observations
    (N), mu (M), sigma^2 (M))."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    F = np.ascontiguousarray(F, dtype=np.float64)
    N, D = X.shape
    K = F.shape[1]
    n0 = N if n0 is None else int(n0)
    W = np.ascontiguousarray(draws, dtype=np.float64).reshape(1 + N - n0, K)
    Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
    M = Xq.shape[0]
    scal, mu, s2 = np.empty(N), np.empty(M), np.empty(M)
    rc = lib.ref_parego(N, n0, D, K, X.ctypes.data, F.ctypes.data, W.ctypes.data, float(rho), float(noise), M, Xq.ctypes.data,
                        scal.ctypes.data, mu.ctypes.data, s2.ctypes.data)
    assert rc == 0, rc
    return scal, mu, s2
