"""Inner optimisers on the hot path's caller side, mirroring src/limbo/opt/:
eval_t helpers (optimizer.hpp:60-96), Rprop (rprop.hpp:82-145) and
ParallelRepeater (parallel_repeater.hpp:76-107), and their lockstep forms BatchedRprop /
BatchedParallelRepeater, which hand every iteration's restarts to the objective at once.
Host control flow only."""
from __future__ import annotations

import math

import numpy as np

from .params import get


def no_grad(x: float):  # optimizer.hpp:66-69
    return (x, None)


def fun(fg) -> float:  # optimizer.hpp:77-81
    return fg[0]


def grad(fg) -> np.ndarray:  # optimizer.hpp:71-75
    assert fg[1] is not None
    return fg[1]


def eval(f, x) -> float:  # optimizer.hpp:84-88
    return f(x, False)[0]


def eval_grad(f, x):  # optimizer.hpp:91-95
    return f(x, True)


def _signum(x: float) -> int:  # tools/math.hpp:71-91
    return int(0 < x) - int(x < 0)


class Rprop:
    def __init__(self, params=None):
        self._params = params

    def __call__(self, f, init, bounded: bool) -> np.ndarray:
        iterations = int(get(self._params, "opt_rprop", "iterations"))
        eps_stop = float(get(self._params, "opt_rprop", "eps_stop"))
        assert eps_stop >= 0.0
        init = np.asarray(init, dtype=np.float64)
        n = init.size
        delta0, deltamin, deltamax, etaminus, etaplus = 0.1, 1e-6, 50.0, 0.5, 1.2
        delta = np.ones(n) * delta0
        grad_old = np.zeros(n)
        params = init.copy()
        if bounded:
            params = np.clip(params, 0.0, 1.0)
        best_params = params.copy()
        best = -math.inf  # log(0)
        for _ in range(iterations):
            perf = eval_grad(f, params)
            lik = fun(perf)
            if lik > best:
                best = lik
                best_params = params.copy()
            g = -np.asarray(grad(perf), dtype=np.float64)
            grad_old = grad_old * g
            for j in range(n):
                if grad_old[j] > 0:
                    delta[j] = min(delta[j] * etaplus, deltamax)
                elif grad_old[j] < 0:
                    delta[j] = max(delta[j] * etaminus, deltamin)
                    g[j] = 0
                params[j] += -_signum(g[j]) * delta[j]
                if bounded and params[j] < 0:
                    params[j] = 0
                if bounded and params[j] > 1:
                    params[j] = 1
            grad_old = g
            if np.linalg.norm(grad_old) < eps_stop:
                break
        return best_params


class ParallelRepeater:
    """Restarts run one after another on the device (each evaluation already fills
    the GPU); multi-GPU runs shard restarts across ranks (limbo_b200.dist)."""

    def __init__(self, params=None, optimizer=None, rng: np.random.Generator | None = None):
        self._params = params
        self._optimizer = optimizer if optimizer is not None else Rprop(params)
        self._rng = rng if rng is not None else np.random.default_rng()

    def __call__(self, f, init, bounded: bool) -> np.ndarray:
        repeats = int(get(self._params, "opt_parallelrepeater", "repeats"))
        epsilon = float(get(self._params, "opt_parallelrepeater", "epsilon"))
        assert repeats > 0
        assert epsilon > 0.0
        init = np.asarray(init, dtype=np.float64)
        best_v, best_val = init, -float(np.finfo(np.float32).max)  # parallel_repeater.hpp:102
        for _ in range(repeats):
            r_deviation = self._rng.random(init.size) * 2.0 * epsilon - epsilon
            v = self._optimizer(f, init + r_deviation, bounded)
            val = eval(f, v)
            if val > best_val:
                best_v, best_val = v, val
        return best_v


def _eval_batch(f, X: np.ndarray, compute_grad: bool):
    """(values (R,), gradients (R x n) or None) of the R rows of X: f.batch when the objective has one, else f row by row."""
    if hasattr(f, "batch"):
        lik, g = f.batch(X, compute_grad)
        return np.asarray(lik, dtype=np.float64), (np.asarray(g, dtype=np.float64) if compute_grad else None)
    vals = np.empty(X.shape[0])
    grads = np.empty(X.shape) if compute_grad else None
    for r in range(X.shape[0]):
        fg = f(X[r].copy(), compute_grad)
        vals[r] = fun(fg)
        if compute_grad:
            grads[r] = grad(fg)
    return vals, grads


class BatchedRprop:
    """Rprop (rprop.hpp:82-145) on R starting points in lockstep: lane r follows exactly the iterates Rprop would from init[r]
    (the best-seen point, the eps_stop break and the bounded clipping per lane), and every iteration evaluates the lanes still
    running in one f.batch(X, True) call.  A lane that has stopped is no longer evaluated.  Returns the R best points."""

    def __init__(self, params=None):
        self._params = params

    def __call__(self, f, init, bounded: bool) -> np.ndarray:
        iterations = int(get(self._params, "opt_rprop", "iterations"))
        eps_stop = float(get(self._params, "opt_rprop", "eps_stop"))
        assert eps_stop >= 0.0
        params = np.array(np.atleast_2d(init), dtype=np.float64)
        R, n = params.shape
        delta0, deltamin, deltamax, etaminus, etaplus = 0.1, 1e-6, 50.0, 0.5, 1.2
        delta = np.full((R, n), delta0)
        grad_old = np.zeros((R, n))
        if bounded:
            params = np.clip(params, 0.0, 1.0)
        best_params = params.copy()
        best = np.full(R, -math.inf)
        live = np.arange(R)
        for _ in range(iterations):
            if live.size == 0:
                break
            lik, gr = _eval_batch(f, params[live].copy(), True)
            better = lik > best[live]  # NaN compares false, as in Rprop
            best[live[better]] = lik[better]
            best_params[live[better]] = params[live[better]]
            g = -gr
            go = grad_old[live] * g
            d = delta[live]
            up, down = go > 0, go < 0
            d = np.where(up, np.minimum(d * etaplus, deltamax), d)
            d = np.where(down, np.maximum(d * etaminus, deltamin), d)
            g = np.where(down, 0.0, g)
            sgn = (g > 0).astype(np.int64) - (g < 0).astype(np.int64)  # tools/math.hpp signum: 0 for NaN
            p = params[live] + (-sgn) * d
            if bounded:
                p = np.where(p < 0, 0.0, p)
                p = np.where(p > 1, 1.0, p)
            params[live], delta[live], grad_old[live] = p, d, g
            keep = np.array([not (np.linalg.norm(grad_old[r]) < eps_stop) for r in live], dtype=bool)
            live = live[keep]
        return best_params


class BatchedParallelRepeater:
    """ParallelRepeater (parallel_repeater.hpp:76-107) with its restarts run in lockstep by BatchedRprop: the R deviations are
    drawn in restart order from the same rng calls, the R searches share every objective evaluation, one batched evaluation
    without gradient scores the R results, and the first strictly larger value wins, from (init, -FLT_MAX) - the point
    ParallelRepeater(Rprop) returns."""

    def __init__(self, params=None, optimizer=None, rng: np.random.Generator | None = None):
        self._params = params
        self._optimizer = optimizer if optimizer is not None else BatchedRprop(params)
        self._rng = rng if rng is not None else np.random.default_rng()

    def __call__(self, f, init, bounded: bool) -> np.ndarray:
        repeats = int(get(self._params, "opt_parallelrepeater", "repeats"))
        epsilon = float(get(self._params, "opt_parallelrepeater", "epsilon"))
        assert repeats > 0
        assert epsilon > 0.0
        init = np.asarray(init, dtype=np.float64)
        starts = np.stack([init + (self._rng.random(init.size) * 2.0 * epsilon - epsilon) for _ in range(repeats)])
        V = self._optimizer(f, starts, bounded)
        vals, _ = _eval_batch(f, V.copy(), False)
        best_v, best_val = init, -float(np.finfo(np.float32).max)  # parallel_repeater.hpp:102
        for r in range(repeats):
            if vals[r] > best_val:
                best_v, best_val = V[r].copy(), vals[r]
        return best_v
