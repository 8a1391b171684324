"""Client-side plumbing of the batched methods of model.GP and model.SPGP: the arrays they hand to the C ABI, the first mean of a
model at the candidates, and the argmax and values-and-gradients calls with their result arrays."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _lib


def ptr(a: np.ndarray | None) -> int | None:
    """The address of a's data, or None (NULL) for None."""
    return None if a is None else a.ctypes.data


def candidates(Xq) -> np.ndarray:
    """The candidates as a row-major M x D fp64 array."""
    return np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)


def acq_param_pair(p) -> np.ndarray:
    """An acquisition's parameters, padded with a 0 when there is one: the library reads two."""
    ap = np.ascontiguousarray(np.atleast_1d(p), dtype=np.float64)
    return np.append(ap, 0.0) if ap.size < 2 else ap


def first_mean(model, Xq):
    """First output of the model's mean functor at every candidate, as (array, 0.0), or (None, constant) for a constant mean."""
    mf = model.mean_function()
    if mf.is_constant():
        return None, float(np.asarray(mf(Xq[0], model))[0])
    return np.ascontiguousarray(mf.batch(Xq, model)[:, 0]), 0.0


def first_mean_and_grad(model, Xq, prior=None):
    """first_mean and the M x D input gradient of the mean's first output, or None where it is 0: (array or None, constant,
    gradient or None).  The gradient comes first, so a mean without one (mean.BaseMean.grad_x) raises NotImplementedError before
    anything else runs; prior(D), when given, runs next, before the mean is evaluated."""
    mgrad = np.ascontiguousarray(model.mean_function().grad_x(Xq, model)[:, 0, :])
    if prior is not None:
        prior(Xq.shape[1])
    mean0, mconst = first_mean(model, Xq)
    return mean0, mconst, (mgrad if np.any(mgrad) else None)


def argmax(lib, name: str, M: int, return_values: bool, *args):
    """Calls lib.<name>(*args, values, &best, &idx), values being M doubles or NULL; returns (best, idx[, values])."""
    vals = np.empty(M) if return_values else None
    best, idx = C.c_double(), C.c_int64()
    _lib.check(getattr(lib, name)(*args, ptr(vals), C.addressof(best), C.addressof(idx)), name)
    return (best.value, idx.value, vals) if return_values else (best.value, idx.value)


def values_and_grads(lib, name: str, M: int, D: int, *args):
    """Calls lib.<name>(*args, values, grads); returns the M values and the M x D gradients."""
    vals, grads = np.empty(M), np.empty((M, D))
    _lib.check(getattr(lib, name)(*args, ptr(vals), ptr(grads)), name)
    return vals, grads


def constant_mean(model, D: int) -> float:
    """The first output of the model's mean functor when it does not depend on the input; NotImplementedError otherwise (a search
    that runs on the device cannot call a host mean at every generation)."""
    mf = model.mean_function()
    if not mf.is_constant():
        raise NotImplementedError("the device CMA-ES takes input-free means only")
    return float(np.asarray(mf(np.zeros(D), model))[0])


def cmaes(lib, name: str, D: int, *args, lam: int = 0, sigma0: float = 0.5, generations: int = 100, tolx: float = 1e-12, seed: int = 0,
          bounded: bool = True):
    """Calls lib.<name>(*args, &opts, R, starts, best_x, &best_val, &n_evals), args ending with the R x D starts; returns
    (best_x, best_val, n_evals)."""
    starts = candidates(args[-1])
    opts = _lib.CmaesOpts(int(lam), float(sigma0), int(generations), float(tolx), int(seed) & 0xFFFFFFFFFFFFFFFF, int(bool(bounded)))
    bx, bv, n = np.empty(D), C.c_double(), C.c_int64()
    _lib.check(getattr(lib, name)(*args[:-1], C.byref(opts), starts.shape[0], ptr(starts), ptr(bx), C.addressof(bv), C.addressof(n)), name)
    return bx, bv.value, n.value
