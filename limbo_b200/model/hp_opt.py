"""Hyper-parameter optimisation functors mirroring src/limbo/model/gp/*.hpp."""
from __future__ import annotations

import sys

import numpy as np

from .. import _lib
from .. import opt as _opt


class HPOpt:  # model/gp/hp_opt.hpp:57-76
    def __init__(self, params=None, optimizer=None):
        self._params = params
        self._optimizer = optimizer if optimizer is not None else _opt.Rprop(params)
        self._called = False


class NoLFOpt(HPOpt):  # model/gp/no_lf_opt.hpp:55-65
    def __call__(self, gp) -> None:
        print("'NoLFOpt' was called: nothing to optimize", file=sys.stderr)


class KernelLFOpt(HPOpt):
    """model/gp/kernel_lf_opt.hpp:57-97: maximise the log marginal likelihood over the
    kernel h-params.  Each evaluation is one device pipeline
    K -> L -> alpha -> log-lik [-> K^-1 -> gradient] on a private copy of the GP."""

    def __call__(self, gp) -> None:
        self._called = True
        optimization = _KernelLFOptimization(gp)
        params = self._optimizer(optimization, gp.kernel_function().h_params(), False)
        gp.kernel_function().set_h_params(params)
        gp.recompute(False)
        gp.compute_log_lik()


def batch_pays(n: int, rows: int) -> bool:
    """Whether one lb_lml_grad_batch call of `rows` vectors at n samples beats `rows` evaluations of the single path: n within
    LB_LML_BATCH_MAX_N, and rows at least (n / 90)^2, the crossover measured on an H100 (DESIGN.md §4.12: one call costs about as
    much as 1 single evaluation at n = 50, 1.5 at n = 100 and 5 at n = 200), so a lone lane left running after eps_stop stopped
    the others goes back to the single path."""
    return n <= _lib.LML_BATCH_MAX_N and rows * 8100 >= n * n


class _KernelLFOptimization:
    def __init__(self, gp):
        self._original_gp = gp
        self._work = None

    def __call__(self, params, compute_grad: bool):
        # kernel_lf_opt.hpp:79: GP gp(this->_original_gp) - a fresh copy per evaluation, like the reference.  lb_clone
        # shares the source's device buffers (copy-on-write) and the refit draws its N x N buffers from the pool, so
        # after the first evaluation this allocates and copies nothing on the device.
        gp = self._original_gp.copy()
        gp.kernel_function().set_h_params(np.asarray(params, dtype=np.float64))
        gp.recompute(False)
        lik = gp.compute_log_lik()
        if not compute_grad:
            return _opt.no_grad(lik)
        return lik, gp.compute_kernel_grad_log_lik()

    def batch(self, X, compute_grad: bool):
        """The R rows of X at once (opt.BatchedRprop, opt.BatchedParallelRepeater): one lb_lml_grad_batch call where it pays
        (batch_pays), otherwise row by row through __call__."""
        X = np.ascontiguousarray(np.atleast_2d(np.asarray(X, dtype=np.float64)))
        if batch_pays(self._original_gp.nb_samples(), X.shape[0]):
            lik, grad, _ = self._original_gp.lml_grad_batch(X, compute_grad)
            return lik, grad
        rows = [self(x, compute_grad) for x in X]
        return np.array([r[0] for r in rows]), (np.stack([r[1] for r in rows]) if compute_grad else None)


class KernelLooOpt(HPOpt):
    """model/gp/kernel_loo_opt.hpp:57-97: maximise the leave-one-out log predictive probability over the kernel
    h-params (lb_log_loo_cv / lb_kernel_grad_log_loo_cv)."""

    def __call__(self, gp) -> None:
        self._called = True
        optimization = _KernelLooOptimization(gp)
        params = self._optimizer(optimization, gp.kernel_function().h_params(), False)
        gp.kernel_function().set_h_params(params)
        gp.recompute(False)
        gp.compute_log_loo_cv()


class _KernelLooOptimization:
    def __init__(self, gp):
        self._original_gp = gp
        self._work = None

    def __call__(self, params, compute_grad: bool):
        gp = self._original_gp.copy()  # kernel_loo_opt.hpp:79 (device buffers shared copy-on-write / pooled)
        gp.kernel_function().set_h_params(np.asarray(params, dtype=np.float64))
        gp.recompute(False)
        loo = gp.compute_log_loo_cv()
        if not compute_grad:
            return _opt.no_grad(loo)
        return loo, gp.compute_kernel_grad_log_loo_cv()


class KernelMeanLFOpt(HPOpt):
    """model/gp/kernel_mean_lf_opt.hpp:57-122: likelihood over [kernel h-params, mean h-params] jointly."""

    def __call__(self, gp) -> None:
        self._called = True
        optimization = _KernelMeanLFOptimization(gp)
        nk = gp.kernel_function().h_params_size()
        init = np.concatenate([gp.kernel_function().h_params(), gp.mean_function().h_params()])
        params = self._optimizer(optimization, init, False)
        gp.kernel_function().set_h_params(params[:nk])
        gp.mean_function().set_h_params(params[nk:])
        gp.recompute(True)
        gp.compute_log_lik()


class _KernelMeanLFOptimization:
    def __init__(self, gp):
        self._original_gp = gp
        self._work = None

    def __call__(self, params, compute_grad: bool):
        if self._work is None:
            self._work = self._original_gp.copy()
        gp = self._work
        params = np.asarray(params, dtype=np.float64)
        nk = gp.kernel_function().h_params_size()
        gp.kernel_function().set_h_params(params[:nk])
        gp.mean_function().set_h_params(params[nk:])
        gp.recompute(True)
        lik = gp.compute_log_lik()
        if not compute_grad:
            return _opt.no_grad(lik)
        return lik, np.concatenate([gp.compute_kernel_grad_log_lik(), gp.compute_mean_grad_log_lik()])


class MeanLFOpt(HPOpt):
    """model/gp/mean_lf_opt.hpp:57-118: likelihood over the mean h-params only; the factor is kept
    (recompute(true, false) = lb_refit_alpha)."""

    def __call__(self, gp) -> None:
        self._called = True
        optimization = _MeanLFOptimization(gp)
        params = self._optimizer(optimization, gp.mean_function().h_params(), False)
        gp.mean_function().set_h_params(params)
        gp.recompute(True, False)
        gp.compute_log_lik()


class _MeanLFOptimization:
    def __init__(self, gp):
        self._work = gp.copy()  # mean_lf_opt.hpp:96-99: own copy with K^-1 precomputed
        self._work.compute_inv_kernel()

    def __call__(self, params, compute_grad: bool):
        gp = self._work
        gp.mean_function().set_h_params(np.asarray(params, dtype=np.float64))
        gp.recompute(True, False)
        lik = gp.compute_log_lik()
        if not compute_grad:
            return _opt.no_grad(lik)
        return lik, gp.compute_mean_grad_log_lik()


class ParallelLFOpt(HPOpt):
    """model/multi_gp/parallel_lf_opt.hpp:57-70: optimise every inner GP of a MultiGP independently with `inner`
    (an HPOpt class, e.g. KernelLFOpt).  The reference fans the loop over tools::par; the inner GPs here are separate
    device handles (own streams), the host loop only enqueues work."""

    def __init__(self, params=None, inner=None, optimizer=None):
        super().__init__(params, optimizer)
        self._inner = inner if inner is not None else NoLFOpt

    def __call__(self, gp) -> None:
        self._called = True
        for g in gp.gp_models():
            self._inner(self._params, self._optimizer)(g)
