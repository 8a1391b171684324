"""Acquisition functions mirroring src/limbo/acqui/{ucb,gp_ucb,ei}.hpp and src/limbo/experimental/acqui/{eci,ehvi}.hpp.  The scalar
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
        if gradient:  # one device call (lb_acq_grad), FirstElem aggregator only
            return _one_point_grad(self, v, afun)
        mu, sigma = self._model.query(v)
        return opt.no_grad(afun(mu) + self._alpha() * math.sqrt(sigma))

    def argmax_batch(self, Xq, return_values: bool = False):
        return self._model.acq_argmax_batch(_lib.ACQ_UCB, [self._alpha(), 0.0], Xq, return_values)

    def grad_batch(self, Xq):
        """values (M) and gradients (M x D) at M candidates in one device pass"""
        return self._model.acq_grad_batch(_lib.ACQ_UCB, [self._alpha(), 0.0], Xq)

    def cmaes_batch(self, starts, **opts):
        """(best_x, best_val, n_evals) of a batched CMA-ES on the device from each row of starts (the model's acq_cmaes_batch:
        model.GP or model.SPGP)"""
        return self._model.acq_cmaes_batch(_lib.ACQ_UCB, [self._alpha(), 0.0], starts, **opts)

    def _col_params(self):
        return [[self._alpha(), 0.0]] * self._model.dim_out()

    def argmax_cols(self, Xq, return_values: bool = False):
        """argmax_batch in each output column of the model from one device query (model.GP.acq_argmax_cols, e.g. the q columns of
        model.GPParego): (best_values (q), best_indices (q)[, values (M x q)])"""
        return self._model.acq_argmax_cols(_lib.ACQ_UCB, self._col_params(), Xq, return_values)

    def cmaes_cols(self, starts, cols, **opts):
        """(best_x (q x D), best_val (q), n_evals) of a batched CMA-ES on the device in which the instance from starts[i] searches
        column cols[i] (model.GP.acq_cmaes_cols)"""
        return self._model.acq_cmaes_cols(_lib.ACQ_UCB, self._col_params(), starts, cols, **opts)


def _one_point_grad(acqui, v, afun):
    assert afun is first_elem
    vals, grads = acqui.grad_batch(np.atleast_2d(np.asarray(v, dtype=np.float64)))
    return float(vals[0]), grads[0]


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
        if gradient:  # one device call (lb_acq_grad), FirstElem aggregator only
            return _one_point_grad(self, v, afun)
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

    def grad_batch(self, Xq):
        """values (M) and gradients (M x D) at M candidates in one device pass; 0 before the model has samples"""
        Xq = np.atleast_2d(Xq)
        if len(self._model.samples()) < 1:
            return np.zeros(len(Xq)), np.zeros(Xq.shape)
        self._update_f_max(first_elem)
        return self._model.acq_grad_batch(_lib.ACQ_EI, [self._f_max, float(get(self._params, "acqui_ei", "jitter"))], Xq)

    def cmaes_batch(self, starts, **opts):
        """(best_x, best_val, n_evals) of a batched CMA-ES on the device from each row of starts (the model's acq_cmaes_batch:
        model.GP or model.SPGP); before the model has samples every value is 0 and the first start is returned"""
        starts = np.atleast_2d(starts)
        if len(self._model.samples()) < 1:
            return np.array(starts[0], dtype=np.float64), 0.0, 0
        self._update_f_max(first_elem)
        return self._model.acq_cmaes_batch(_lib.ACQ_EI, [self._f_max, float(get(self._params, "acqui_ei", "jitter"))], starts, **opts)

    def _col_params(self):
        """per column: f_max = max_i mu_r(x_i) over the samples (ei.hpp:100-108 with the column's element), from one N-point query of
        every column, and the jitter"""
        mu, _ = self._model.query_batch(np.stack(self._model.samples(), axis=0))
        jitter = float(get(self._params, "acqui_ei", "jitter"))
        return [[float(f), jitter] for f in mu.max(axis=0)]

    def argmax_cols(self, Xq, return_values: bool = False):
        """argmax_batch in each output column of the model from one device query (UCB.argmax_cols); 0 everywhere, index 0, before
        the model has samples"""
        q = self._model.dim_out()
        if len(self._model.samples()) < 1:
            vals = np.zeros((len(Xq), q))
            return (np.zeros(q), np.zeros(q, dtype=np.int64), vals) if return_values else (np.zeros(q), np.zeros(q, dtype=np.int64))
        return self._model.acq_argmax_cols(_lib.ACQ_EI, self._col_params(), Xq, return_values)

    def cmaes_cols(self, starts, cols, **opts):
        """UCB.cmaes_cols over EI; before the model has samples every value is 0 and each column returns its first start"""
        starts = np.atleast_2d(starts)
        if len(self._model.samples()) < 1:
            cols = np.asarray(cols)
            q = self._model.dim_out()
            return np.stack([starts[int(np.argmax(cols == r))] for r in range(q)]).astype(np.float64), np.zeros(q), 0
        return self._model.acq_cmaes_cols(_lib.ACQ_EI, self._col_params(), starts, cols, **opts)


class ECI(_Improvement):
    """Expected constrained improvement (experimental/acqui/eci.hpp): EI on `model` weighted by the probability Pf that the first
    output of `constraint_model` exceeds 1.  Pf = 1 when the constraint model has no samples or is None.  Both models are
    model.GP; argmax_batch, grad_batch and cmaes_batch each run in one device call over both."""

    def __init__(self, model, constraint_model, iteration: int = 0, params=None):
        super().__init__(model, params)
        self._constraint_model = constraint_model

    def _jitter(self) -> float:
        return float(get(self._params, "acqui_eci", "jitter"))

    def __call__(self, v, afun=first_elem, gradient: bool = False):  # eci.hpp:76-107
        if gradient:  # one device call (lb_eci_grad), FirstElem aggregator only
            return _one_point_grad(self, v, afun)
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

    def grad_batch(self, Xq):
        """values (M) and gradients (M x D) at M candidates in one device pass over both models; 0 before the objective has samples"""
        Xq = np.atleast_2d(Xq)
        if len(self._model.samples()) < 1:
            return np.zeros(len(Xq)), np.zeros(Xq.shape)
        self._update_f_max(first_elem)
        return self._model.eci_grad_batch(self._constraint_model, self._f_max, self._jitter(), Xq)

    def cmaes_batch(self, starts, **opts):
        """(best_x, best_val, n_evals) of a batched CMA-ES on the device from each row of starts, over both models
        (model.GP.eci_cmaes_batch); before the objective has samples every value is 0 and the first start is returned"""
        starts = np.atleast_2d(starts)
        if len(self._model.samples()) < 1:
            return np.array(starts[0], dtype=np.float64), 0.0, 0
        self._update_f_max(first_elem)
        return self._model.eci_cmaes_batch(self._constraint_model, self._f_max, self._jitter(), starts, **opts)


class EHVI:
    """Expected hypervolume improvement over two or three objectives (experimental/acqui/ehvi.hpp): `models` are the objectives'
    GPs, `pop` the k x 2 (k x 3) objective values of the current Pareto front (the reference's deque of individuals), `ref_point`
    the reference point (its first two (three) entries are used).  As in the reference, each model's sigma() (sigma^2 + noise) is
    passed where ehvi2d / ehvi3d_sliceupdate expect a standard deviation.  Every evaluation, the one-point __call__ included, runs
    on the device (lb_ehvi_argmax or lb_ehvi3d_argmax, and lb_ehvi_grad for two-objective gradients; three-objective gradients
    raise NotImplementedError).  cmaes_batch searches two or three objectives (lb_ehvi_cmaes); the models are model.GP."""

    def __init__(self, models, pop, ref_point, params=None):
        assert len(models) in (2, 3)  # ehvi.hpp:65 (two); three run ehvi3d_sliceupdate
        self._models, self._params = models, params
        K = len(models)
        self._pop = np.ascontiguousarray(np.asarray(pop, dtype=np.float64).reshape(-1, K))
        self._ref_point = np.asarray(ref_point, dtype=np.float64).reshape(-1)[:K].copy()

    def dim_in(self):
        return self._models[0].dim_in()

    def dim_out(self):
        return 1

    def __call__(self, v, afun=first_elem, gradient: bool = False):  # ehvi.hpp:70-79, FirstElem aggregator only
        assert afun is first_elem
        if gradient:  # one device call (lb_ehvi_grad)
            return _one_point_grad(self, v, afun)
        best, _ = self.argmax_batch(np.atleast_2d(np.asarray(v, dtype=np.float64)))
        return opt.no_grad(best)

    def argmax_batch(self, Xq, return_values: bool = False):
        if len(self._models) == 3:
            return self._models[0].ehvi3d_argmax_batch(self._models[1], self._models[2], self._ref_point, self._pop, Xq, return_values)
        return self._models[0].ehvi_argmax_batch(self._models[1], self._ref_point, self._pop, Xq, return_values)

    def grad_batch(self, Xq):
        """values (M) and gradients (M x D) at M candidates in one device pass over both models (two objectives only)"""
        if len(self._models) == 3:
            raise NotImplementedError("the three-objective EHVI has no gradient on the device")
        return self._models[0].ehvi_grad_batch(self._models[1], self._ref_point, self._pop, Xq)

    def cmaes_batch(self, starts, **opts):
        """(best_x, best_val, n_evals) of a batched CMA-ES on the device from each row of starts, over two or three objectives
        (model.GP.ehvi_cmaes_batch)"""
        return self._models[0].ehvi_cmaes_batch(self._models[1:], self._ref_point, self._pop, starts, **opts)
