"""The outer loop that drives the hot path, mirroring bayes_opt::BOptimizer::optimize
(src/limbo/bayes_opt/boptimizer.hpp:139-170, bo_base.hpp:220-283) with a device-aware inner acquisition
optimiser: the reference's optimisers evaluate one point at a time (opt/optimizer.hpp:84-96), which would leave the GPU
idle; `BatchedRandomSearch` scores a whole candidate set per call through lb_acq_argmax (SURVEY.md §8f rank 2)."""
from __future__ import annotations

import numpy as np

from . import acqui as _acqui
from .params import get


class defaults_bo:
    class init_randomsampling:  # init/random_sampling.hpp:57-60
        samples = 10

    class stop_maxiterations:  # stop/max_iterations.hpp:56-59
        iterations = 190

    class opt_batchedrandom:
        candidates = 20000
        refinements = 2
        shrink = 0.1


def _get(params, section, name):
    sec = getattr(params, section, None) if params is not None else None
    if sec is not None and hasattr(sec, name):
        return getattr(sec, name)
    return getattr(getattr(defaults_bo, section), name)


class EvaluationError(Exception):  # bo_base.hpp:106-107
    pass


class BatchedRandomSearch:
    """acquiopt<> policy: uniform candidates in [0,1]^D scored in one device pass, then `refinements` rounds of
    candidates drawn in a box shrinking around the incumbent."""

    def __init__(self, params=None, rng: np.random.Generator | None = None):
        self._params = params
        self._rng = rng if rng is not None else np.random.default_rng()

    def __call__(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        m = int(_get(self._params, "opt_batchedrandom", "candidates"))
        cand = self._rng.random((m, dim))
        best, idx = acqui.argmax_batch(cand)
        x = cand[idx].copy()
        radius = 1.0
        for _ in range(int(_get(self._params, "opt_batchedrandom", "refinements"))):
            radius *= float(_get(self._params, "opt_batchedrandom", "shrink"))
            cand = x + (self._rng.random((m, dim)) * 2.0 - 1.0) * radius
            if bounded:
                cand = np.clip(cand, 0.0, 1.0)
            cand[0] = x  # keep the incumbent in the set
            b2, i2 = acqui.argmax_batch(cand)
            if b2 >= best:
                best, x = b2, cand[i2].copy()
        return x


class BOptimizer:
    def __init__(self, model, params=None, acqui=_acqui.UCB, acqui_opt=None, rng: np.random.Generator | None = None):
        self._model, self._params, self._acqui_cls = model, params, acqui
        self._rng = rng if rng is not None else np.random.default_rng()
        self._acqui_opt = acqui_opt if acqui_opt is not None else BatchedRandomSearch(params, self._rng)
        self._samples: list[np.ndarray] = []
        self._observations: list[np.ndarray] = []
        self._current_iteration = 0
        self._total_iterations = 0

    # bo_base.hpp:220-245
    def add_new_sample(self, s, v) -> None:
        self._samples.append(np.asarray(s, dtype=np.float64))
        self._observations.append(np.atleast_1d(np.asarray(v, dtype=np.float64)))

    def eval_and_add(self, sfun, sample) -> None:
        v = np.atleast_1d(np.asarray(sfun(sample), dtype=np.float64))
        if np.any(~np.isfinite(v)):
            raise EvaluationError("the evaluation function returned NaN or inf")
        self.add_new_sample(sample, v)

    def optimize(self, sfun, dim_in: int, afun=_acqui.first_elem, reset: bool = True) -> None:
        # boptimizer.hpp:139-170
        if reset:
            self._samples, self._observations = [], []
            self._current_iteration = 0
        if self._total_iterations == 0 or reset:
            for _ in range(int(_get(self._params, "init_randomsampling", "samples"))):  # init/random_sampling.hpp:73-79
                self.eval_and_add(sfun, self._rng.random(dim_in))
        if self._observations:
            self._model.compute(np.stack(self._samples), np.stack(self._observations))
        hp_period = int(get(self._params, "bayes_opt_boptimizer", "hp_period"))
        max_it = int(_get(self._params, "stop_maxiterations", "iterations"))
        while self._current_iteration < max_it:
            acqui = self._acqui_cls(self._model, self._current_iteration, params=self._params)
            x = self._acqui_opt(acqui, dim_in, True)
            self.eval_and_add(sfun, x)
            self._model.add_sample(self._samples[-1], self._observations[-1])
            if hp_period > 0 and (self._current_iteration + 1) % hp_period == 0:
                self._model.optimize_hyperparams()
            self._current_iteration += 1
            self._total_iterations += 1

    def best_observation(self, afun=_acqui.first_elem) -> np.ndarray:  # boptimizer.hpp:173-180
        return max(self._observations, key=afun)

    def best_sample(self, afun=_acqui.first_elem) -> np.ndarray:  # boptimizer.hpp:183-190
        i = int(np.argmax([afun(o) for o in self._observations]))
        return self._samples[i]

    def model(self):
        return self._model

    def samples(self):
        return self._samples

    def observations(self):
        return self._observations


class CBOptimizer(BOptimizer):
    """Constrained Bayesian optimisation, mirroring experimental::bayes_opt::CBOptimizer
    (src/limbo/experimental/bayes_opt/cboptimizer.hpp:149-260).  Every observation holds `dim_out` objective values followed
    by `nb_constraints` constraint values; an observation is feasible when the product of its constraint values is > 0.  The
    objective model and a constraint model (default: GP(dim_in, nb_constraints, kernel=Exp, mean=Constant)) are both updated
    every iteration, and the acquisition (default acqui.ECI) is built over the pair.

    Three deliberate deviations from the reference:
      (a) the new observation is split into its objective and constraint parts every iteration before add_sample; the
          reference adds ``_obs[0].back()`` (cboptimizer.hpp:181), which is stale unless something called best_observation();
      (b) best_sample() returns the sample paired with the best feasible observation; the reference indexes the samples with
          the position in the feasible-only list (cboptimizer.hpp:228);
      (c) with nb_constraints == 0 every observation is feasible; the reference indexes an empty constraint list
          (cboptimizer.hpp:244)."""

    def __init__(self, model, constraint_model=None, params=None, acqui=_acqui.ECI, acqui_opt=None,
                 rng: np.random.Generator | None = None):
        super().__init__(model, params, acqui, acqui_opt, rng)
        self._constraint_model = constraint_model
        self._dim_out, self._nb_constraints = 1, 0

    def _split(self, observation) -> tuple[np.ndarray, np.ndarray]:  # cboptimizer.hpp:251-272
        o = np.asarray(observation, dtype=np.float64)
        assert o.size == self._dim_out + self._nb_constraints
        return o[: self._dim_out], o[self._dim_out:]

    def optimize(self, sfun, dim_in: int, dim_out: int = 1, nb_constraints: int = 0, afun=_acqui.first_elem,
                 reset: bool = True) -> None:
        # cboptimizer.hpp:149-192
        self._dim_out, self._nb_constraints = int(dim_out), int(nb_constraints)
        if self._constraint_model is None and self._nb_constraints > 0:
            from . import kernel as _kernel, mean as _mean
            from .model import GP
            self._constraint_model = GP(dim_in, self._nb_constraints, params=self._params, kernel=_kernel.Exp, mean=_mean.Constant)
        if reset:
            self._samples, self._observations = [], []
            self._current_iteration = 0
        if self._total_iterations == 0 or reset:
            for _ in range(int(_get(self._params, "init_randomsampling", "samples"))):
                self.eval_and_add(sfun, self._rng.random(dim_in))
        if self._observations:
            parts = [self._split(o) for o in self._observations]
            self._model.compute(np.stack(self._samples), np.stack([p[0] for p in parts]))
            if self._nb_constraints > 0:
                self._constraint_model.compute(np.stack(self._samples), np.stack([p[1] for p in parts]))
        con = self._constraint_model if self._nb_constraints > 0 else None
        hp_period = int(get(self._params, "bayes_opt_cboptimizer", "hp_period"))
        bounded = bool(get(self._params, "bayes_opt_cboptimizer", "bounded"))
        max_it = int(_get(self._params, "stop_maxiterations", "iterations"))
        while self._current_iteration < max_it:
            acqui = self._acqui_cls(self._model, con, self._current_iteration, params=self._params)
            x = self._acqui_opt(acqui, dim_in, bounded)
            self.eval_and_add(sfun, x)
            obj, cons = self._split(self._observations[-1])  # deviation (a)
            self._model.add_sample(self._samples[-1], obj)
            if con is not None:
                con.add_sample(self._samples[-1], cons)
            if hp_period > 0 and (self._current_iteration + 1) % hp_period == 0:
                self._model.optimize_hyperparams()
                if con is not None:
                    con.optimize_hyperparams()
            self._current_iteration += 1
            self._total_iterations += 1

    def _best_index(self, afun) -> int:  # cboptimizer.hpp:197-248, deviations (b) and (c)
        parts = [self._split(o) for o in self._observations]
        feasible = [i for i, (_, c) in enumerate(parts) if np.prod(c) > 0]  # prod of no constraints = 1
        candidates = feasible if feasible else list(range(len(parts)))
        return max(candidates, key=lambda i: afun(parts[i][0]))  # the first maximum, as std::max_element

    def best_observation(self, afun=_acqui.first_elem) -> np.ndarray:
        return self._split(self._observations[self._best_index(afun)])[0]

    def best_sample(self, afun=_acqui.first_elem) -> np.ndarray:
        return self._samples[self._best_index(afun)]

    def constraint_model(self):
        return self._constraint_model
