"""ctypes front-end of oracle/_ref/libref_sparse.so: the reference's OWN model::SparsifiedGP::_sparsify
(oracle/ref_shim/sparse_driver.cpp, built by oracle/ref_shim/Makefile).  TEST INFRASTRUCTURE ONLY; built only where the
reference's sources are present (oracle/ref.py: REF_SRC) — elsewhere the tests rely on tests/golden/sparsify/."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .ref import RefLibrary


def _declare(lib):
    vp, lg, i = C.c_void_p, C.c_long, C.c_int
    lib.ref_sparsify.argtypes = [lg, i, vp, lg] + [vp] * 5
    lib.ref_sparsify.restype = i


_LIB = RefLibrary("libref_sparse.so", _declare)
LIB_PATH, available, load = _LIB.path, _LIB.available, _LIB.load


def sparsify(X, max_points: int):
    """The reference's _sparsify on the rows of X.  Returns (kept, removed, removed_score): kept original indices (ascending),
    the removal order and the density min_dist each removed point had when _get_most_dense_point chose it."""
    lib = load()
    X = np.ascontiguousarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X[:, None]
    N, D = X.shape
    kept = np.empty(N, dtype=np.int64)
    removed = np.empty(N, dtype=np.int64)
    score = np.empty(N)
    nk, nr = C.c_long(), C.c_long()
    rc = lib.ref_sparsify(N, D, X.ctypes.data, int(max_points), kept.ctypes.data, C.addressof(nk), removed.ctypes.data, score.ctypes.data,
                          C.addressof(nr))
    assert rc == 0, rc
    return kept[:nk.value].copy(), removed[:nr.value].copy(), score[:nr.value].copy()
