"""Acquisition functions mirroring src/limbo/acqui/{ucb,gp_ucb,ei}.hpp and src/limbo/experimental/acqui/eci.hpp.  The scalar
``__call__(v, afun, gradient)`` keeps the reference contract (one point, any host
aggregator); ``argmax_batch`` is the batched device path (FirstElem aggregator)."""
from __future__ import annotations

import math

import numpy as np

from . import _lib, opt
from .params import get


def first_elem(x):  # bayes_opt/bo_base.hpp:99-105
    return float(np.asarray(x)[0])


class UCB:
    def __init__(self, model, iteration: int = 0, params=None):
        self._model, self._params = model, params

    def dim_in(self):
        return self._model.dim_in()

    def dim_out(self):
        return self._model.dim_out()

    def _alpha(self) -> float:
        return float(get(self._params, "acqui_ucb", "alpha"))

    def __call__(self, v, afun=first_elem, gradient: bool = False):  # ucb.hpp:83-90
        assert not gradient
        mu, sigma = self._model.query(v)
        return opt.no_grad(afun(mu) + self._alpha() * math.sqrt(sigma))

    def argmax_batch(self, Xq, return_values: bool = False):
        return self._model.acq_argmax_batch(_lib.ACQ_UCB, [self._alpha(), 0.0], Xq, return_values)


class GP_UCB(UCB):
    def __init__(self, model, iteration: int, params=None):  # gp_ucb.hpp:83-88
        super().__init__(model, iteration, params)
        nt = math.pow(iteration, model.dim_in() / 2.0 + 2.0)
        delta3 = float(get(params, "acqui_gpucb", "delta")) * 3
        self._beta = math.sqrt(2.0 * math.log(nt * math.pi * math.pi / delta3))

    def _alpha(self) -> float:
        return self._beta


class _Improvement:
    """What EI and ECI share: the objective model and f_max = max_i afun(mu(x_i)) over its samples."""

    def __init__(self, model, params=None):
        self._model, self._params = model, params
        self._nb_samples = -1
        self._f_max = 0.0

    def dim_in(self):
        return self._model.dim_in()

    def dim_out(self):
        return self._model.dim_out()

    def _update_f_max(self, afun) -> None:  # ei.hpp:100-108, eci.hpp:91-99; batched: N mu() calls in one pass
        if self._nb_samples != self._model.nb_samples():
            mu, _ = self._model.query_batch(np.stack(self._model.samples(), axis=0))
            self._f_max = max(afun(m) for m in mu)
            self._nb_samples = self._model.nb_samples()


class EI(_Improvement):
    def __init__(self, model, iteration: int = 0, params=None):
        super().__init__(model, params)

    def __call__(self, v, afun=first_elem, gradient: bool = False):  # ei.hpp:85-116
        assert not gradient
        mu, sigma_sq = self._model.query(v)
        sigma = math.sqrt(sigma_sq)
        if sigma < 1e-10 or len(self._model.samples()) < 1:
            return opt.no_grad(0.0)
        self._update_f_max(afun)
        X = afun(mu) - self._f_max - float(get(self._params, "acqui_ei", "jitter"))
        Z = X / sigma
        phi = math.exp(-0.5 * math.pow(Z, 2.0)) / math.sqrt(2.0 * math.pi)
        Phi = 0.5 * math.erfc(-Z / math.sqrt(2))
        return opt.no_grad(X * Phi + sigma * phi)

    def argmax_batch(self, Xq, return_values: bool = False):
        if len(self._model.samples()) < 1:
            vals = np.zeros(len(Xq))
            return (0.0, 0, vals) if return_values else (0.0, 0)
        self._update_f_max(first_elem)
        return self._model.acq_argmax_batch(_lib.ACQ_EI, [self._f_max, float(get(self._params, "acqui_ei", "jitter"))], Xq,
                                            return_values)


class ECI(_Improvement):
    """Expected constrained improvement (experimental/acqui/eci.hpp): EI on `model` weighted by the probability Pf that the first
    output of `constraint_model` exceeds 1.  Pf = 1 when the constraint model has no samples or is None."""

    def __init__(self, model, constraint_model, iteration: int = 0, params=None):
        super().__init__(model, params)
        self._constraint_model = constraint_model

    def _jitter(self) -> float:
        return float(get(self._params, "acqui_eci", "jitter"))

    def __call__(self, v, afun=first_elem, gradient: bool = False):  # eci.hpp:76-107
        assert not gradient
        mu, sigma_sq = self._model.query(v)
        sigma = math.sqrt(sigma_sq)
        if sigma < 1e-10 or len(self._model.samples()) < 1:
            return opt.no_grad(0.0)
        self._update_f_max(afun)
        X = afun(mu) - self._f_max - self._jitter()
        Z = X / sigma
        phi = math.exp(-0.5 * math.pow(Z, 2.0)) / math.sqrt(2.0 * math.pi)
        Phi = 0.5 * math.erfc(-Z / math.sqrt(2))
        return opt.no_grad(self._pf(v, afun) * (X * Phi + sigma * phi))

    def _pf(self, v, afun) -> float:  # eci.hpp:116-130
        if self._constraint_model is None:
            return 1.0
        mu, sigma_sq = self._constraint_model.query(v)
        sigma = math.sqrt(sigma_sq)
        if sigma < 1e-10 or len(self._constraint_model.samples()) < 1:
            return 1.0
        Z = (afun(mu) - 1.0) / sigma
        return 0.5 * math.erfc(-Z / math.sqrt(2))

    def argmax_batch(self, Xq, return_values: bool = False):
        if len(self._model.samples()) < 1:
            vals = np.zeros(len(Xq))
            return (0.0, 0, vals) if return_values else (0.0, 0)
        self._update_f_max(first_elem)
        return self._model.eci_argmax_batch(self._constraint_model, self._f_max, self._jitter(), Xq, return_values)
