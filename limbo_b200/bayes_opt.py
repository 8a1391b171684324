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

    class opt_batchedgradient:  # DESIGN.md §4.10 gives the measurement behind these
        candidates = 10000
        starts = 32
        iterations = 30
        alpha = 0.01

    class opt_batchedcmaes:  # DESIGN.md §4.15 gives the measurement behind these
        candidates = 10000
        starts = 32
        # "lambda" is a Python keyword: read with getattr
        sigma = 0.1
        generations = 50
        tolx = 1e-6

setattr(defaults_bo.opt_batchedcmaes, "lambda", 0)


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

    def propose_batch(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        """one point per output column of the acquisition's model (q x D): the column's best of `candidates` uniform points, all
        scored in one device query (the acquisition's argmax_cols); no refinement rounds"""
        cand = self._rng.random((int(_get(self._params, "opt_batchedrandom", "candidates")), dim))
        _, idx = acqui.argmax_cols(cand)
        return cand[np.asarray(idx)].copy()


def _best_distinct(cand, vals, n: int) -> np.ndarray:
    """the (at most) n best distinct rows of cand by vals, descending, NaN last"""
    order = np.argsort(-np.nan_to_num(np.asarray(vals), nan=-np.inf), kind="stable")
    chosen, seen = [], set()
    for i in order:
        key = cand[i].tobytes()
        if key not in seen:
            seen.add(key)
            chosen.append(i)
        if len(chosen) == n:
            break
    return cand[chosen].copy()


class BatchedGradientSearch:
    """acquiopt<> policy: one random pass of `candidates` uniform points in [0,1]^D scored in one device pass, then the best
    `starts` distinct points climb the acquisition in lockstep for `iterations` steps of Adam with the reference's update
    (opt/adam.hpp: b1 = 0.9, b2 = 0.999, epsilon = 1e-8, step `alpha`, clipped to [0, 1] when bounded), each step one batched
    value-and-gradient call (the acquisition's grad_batch) for all starts.  Returns the best point seen, the random pass included;
    with an acquisition that has no grad_batch, or whose model or mean gives no candidate gradient, the best point of the random
    pass."""

    B1, B2, EPS = 0.9, 0.999, 1e-8

    def __init__(self, params=None, rng: np.random.Generator | None = None):
        self._params = params
        self._rng = rng if rng is not None else np.random.default_rng()

    def _p(self, name):
        return _get(self._params, "opt_batchedgradient", name)

    def __call__(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        cand = self._rng.random((int(self._p("candidates")), dim))
        best, idx, vals = acqui.argmax_batch(cand, return_values=True)
        x_best = cand[idx].copy()
        grad_batch = getattr(acqui, "grad_batch", None)
        if grad_batch is None:
            return x_best
        x = _best_distinct(cand, vals, int(self._p("starts")))
        alpha = float(self._p("alpha"))
        m, v = np.zeros_like(x), np.zeros_like(x)
        b1_t, b2_t = self.B1, self.B2
        for it in range(int(self._p("iterations"))):
            try:
                f, g = grad_batch(x)
            except (AttributeError, NotImplementedError):
                # a model without candidate gradients (model.MultiGP) or a mean without an input gradient
                if it == 0:
                    return x_best
                raise
            f = np.nan_to_num(np.asarray(f, dtype=np.float64), nan=-np.inf)
            j = int(np.argmax(f))
            if f[j] > best:
                best, x_best = float(f[j]), x[j].copy()
            m = self.B1 * m + (1.0 - self.B1) * g
            v = self.B2 * v + (1.0 - self.B2) * g * g
            x = x + alpha * (m / (1.0 - b1_t)) / (np.sqrt(v / (1.0 - b2_t)) + self.EPS)
            if bounded:
                x = np.clip(x, 0.0, 1.0)
            b1_t *= self.B1
            b2_t *= self.B2
        return x_best

    def propose_batch(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        raise NotImplementedError("candidate gradients cover the first output column only")


class BatchedCmaesSearch:
    """acquiopt<> policy: one random pass of `candidates` uniform points in [0,1]^D scored in one device pass, then one batched
    CMA-ES on the device (the acquisition's cmaes_batch, DESIGN.md §4.15) with one instance from each of the best `starts`
    distinct points: `lambda` offspring per instance (0: 4 + floor(3 ln D)), initial step `sigma`, at most `generations`
    generations, an instance stopping when sigma sqrt(max diag C) < `tolx`.  The search takes UCB / GP_UCB / EI over model.GP and
    model.SPGP, ECI over an objective and a constraint model.GP, and two- and three-objective EHVI over model.GP.  Returns the
    better of the search's best point and the random pass's (the random pass on ties); with an acquisition that has no
    cmaes_batch, or a model or mean the device search does not take (model.MultiGP, an SPGP before its first compute, a mean that
    depends on the input), the best point of the random pass."""

    def __init__(self, params=None, rng: np.random.Generator | None = None):
        self._params = params
        self._rng = rng if rng is not None else np.random.default_rng()

    def _p(self, name):
        return _get(self._params, "opt_batchedcmaes", name)

    def __call__(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        cand = self._rng.random((int(self._p("candidates")), dim))
        best, idx, vals = acqui.argmax_batch(cand, return_values=True)
        x_best = cand[idx].copy()
        cmaes_batch = getattr(acqui, "cmaes_batch", None)
        if cmaes_batch is None:
            return x_best
        starts = _best_distinct(cand, vals, int(self._p("starts")))
        try:
            x, v, _ = cmaes_batch(starts, lam=int(self._p("lambda")), sigma0=float(self._p("sigma")),
                                  generations=int(self._p("generations")), tolx=float(self._p("tolx")),
                                  seed=int(self._rng.integers(0, 2**63 - 1)), bounded=bounded)
        except (AttributeError, NotImplementedError):
            return x_best
        return np.asarray(x, dtype=np.float64) if v > best else x_best

    def propose_batch(self, acqui, dim: int, bounded: bool = True) -> np.ndarray:
        """one point per output column of the acquisition's model (q x D): one random pass scored in every column at once
        (argmax_cols), then one device CMA-ES (cmaes_cols) with max(1, starts // q) instances per column, started from that column's
        best distinct points; per column the better of the search's point and the random pass's (the random pass on ties)"""
        cand = self._rng.random((int(self._p("candidates")), dim))
        best, idx, vals = acqui.argmax_cols(cand, return_values=True)
        x_best = cand[np.asarray(idx)].copy()
        q = x_best.shape[0]
        per = max(1, int(self._p("starts")) // q)
        starts, cols = [], []
        for r in range(q):
            s = _best_distinct(cand, vals[:, r], per)
            starts.append(s)
            cols += [r] * s.shape[0]
        x, v, _ = acqui.cmaes_cols(np.concatenate(starts), cols, lam=int(self._p("lambda")), sigma0=float(self._p("sigma")),
                                   generations=int(self._p("generations")), tolx=float(self._p("tolx")),
                                   seed=int(self._rng.integers(0, 2**63 - 1)), bounded=bounded)
        better = np.asarray(v) > np.asarray(best)
        x_best[better] = np.asarray(x, dtype=np.float64)[better]
        return x_best


def distinct_rows(X) -> np.ndarray:
    """the rows of X without any row equal to an earlier one, in order"""
    seen, keep = set(), []
    for i, x in enumerate(np.asarray(X, dtype=np.float64)):
        key = x.tobytes()
        if key not in seen:
            seen.add(key)
            keep.append(i)
    return np.asarray(X, dtype=np.float64)[keep]


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


class BoMulti(BOptimizer):
    """Multi-objective base, mirroring experimental::bayes_opt::BoMulti (src/limbo/experimental/bayes_opt/bo_multi.hpp:153-246):
    one GP(dim_in, 1) per objective (kernel and mean as given, Matern-5/2 and mean::Data by default, hyper-parameters from the
    params), refitted from scratch by _update_models, and the Pareto set of the data.  Without sferes' NSGA-II,
    update_pareto_model only refits the models and pareto_model() stays empty, as the reference behaves without USE_SFERES."""

    def __init__(self, params=None, kernel=None, mean=None, acqui=_acqui.EHVI, acqui_opt=None, rng: np.random.Generator | None = None,
                 device: int = 0):
        super().__init__(None, params, acqui, acqui_opt, rng)
        from . import kernel as _kernel, mean as _mean
        self._kernel = kernel if kernel is not None else _kernel.MaternFiveHalves
        self._mean = mean if mean is not None else _mean.Data
        self._device = device
        self._models: list = []
        self._pareto_model: list = []
        self._pareto_data: list = []

    def nb_objs(self) -> int:  # bo_multi.hpp:164
        return int(self._observations[0].size)

    def models(self):
        return self._models

    def pareto_model(self):
        return self._pareto_model

    def pareto_data(self):
        return self._pareto_data

    def update_pareto_data(self) -> None:  # bo_multi.hpp:173-180
        from . import pareto
        zeros = [np.zeros(self.nb_objs())] * len(self._samples)
        self._pareto_data = pareto.pareto_set(self._pack_data(self._samples, self._observations, zeros), 1, self._device)

    def update_pareto_model(self) -> None:  # bo_multi.hpp:183-213 without USE_SFERES
        self._update_models()

    @staticmethod
    def _pack_data(points, objs, sigma) -> list:  # bo_multi.hpp:220-231
        assert len(points) == len(objs) and len(sigma) == len(objs)
        return list(zip(points, objs, sigma))

    def _update_models(self) -> None:  # bo_multi.hpp:233-245: new models every call
        from .model import GP
        dim = self._samples[0].size
        X = np.stack(self._samples)
        Y = np.stack(self._observations)
        self._models = [GP(dim, 1, params=self._params, kernel=self._kernel, mean=self._mean, device=self._device)
                        for _ in range(self.nb_objs())]
        for i, m in enumerate(self._models):
            m.compute(X, Y[:, i:i + 1])


class Ehvi(BoMulti):
    """EHVI-driven multi-objective optimisation, mirroring experimental::bayes_opt::Ehvi
    (src/limbo/experimental/bayes_opt/ehvi.hpp:82-163), over two objectives with reference point (bayes_opt_ehvi.x_ref, y_ref), or
    over three with (x_ref, y_ref, z_ref) and the device's ehvi3d_sliceupdate (the reference's loop stays two-objective).  With three
    objectives the data's Pareto set may hold at most LB_EHVI3D_MAX_K = 256 points: past that, lb_ehvi3d_argmax returns
    LB_ERR_UNSUPPORTED and the iteration raises (with three objectives a front that size comes within a few hundred samples).

    One deliberate deviation: the reference starts one inner optimisation from each point of the data's Pareto set and keeps the
    best (ehvi.hpp:131-147); here every iteration runs one acquisition optimiser (BatchedRandomSearch by default) over [0, 1]^D,
    which scores its whole candidate set in one device pass, as BOptimizer does."""

    def optimize(self, sfun, dim_in: int, reset: bool = True) -> None:
        if reset:
            self._samples, self._observations = [], []
            self._current_iteration = 0
        if self._total_iterations == 0 or reset:
            for _ in range(int(_get(self._params, "init_randomsampling", "samples"))):
                self.eval_and_add(sfun, self._rng.random(dim_in))
        ref = (float(get(self._params, "bayes_opt_ehvi", "x_ref")), float(get(self._params, "bayes_opt_ehvi", "y_ref")))
        max_it = int(_get(self._params, "stop_maxiterations", "iterations"))
        while self._current_iteration < max_it:
            K = self.nb_objs()
            assert K in (2, 3)  # acqui/ehvi.hpp:65, 73; three objectives through ehvi3d_sliceupdate
            r = ref if K == 2 else ref + (float(get(self._params, "bayes_opt_ehvi", "z_ref")),)
            self.update_pareto_model()
            self.update_pareto_data()
            pop = np.array([np.asarray(p[1], dtype=np.float64)[:K] for p in self._pareto_data]).reshape(-1, K)
            acqui = self._acqui_cls(self._models, pop, r, params=self._params)
            x = self._acqui_opt(acqui, dim_in, True)
            self.eval_and_add(sfun, x)
            self._current_iteration += 1
            self._total_iterations += 1


class Parego(BOptimizer):
    """ParEGO, mirroring experimental::bayes_opt::Parego (src/limbo/experimental/bayes_opt/parego.hpp:73-86): BOptimizer over a
    model.GPParego that scalarises the K objectives with random weights (kernel and mean as given, Matern-5/2 and mean::Data by
    default), with a single-output acquisition (UCB by default) and FirstElem.  best_observation() ranks the raw observations, as
    the reference does.

    With q = 1 it is BOptimizer over GPParego, and every acquisition optimiser works.  With q > 1 (qParEGO) the model holds q
    scalarisations, each iteration proposes one point per column through the optimiser's propose_batch (BatchedRandomSearch: one
    argmax_cols over its candidate set; BatchedCmaesSearch: cmaes_cols; BatchedGradientSearch raises NotImplementedError), a
    proposal equal to an earlier column's is dropped, and each evaluated point is one iteration of stop_maxiterations, added with
    its own add_sample (fresh weights each time).  DESIGN.md §4.16."""

    def __init__(self, params=None, q: int = 1, kernel=None, mean=None, acqui=_acqui.UCB, acqui_opt=None,
                 rng: np.random.Generator | None = None, device: int = 0, hp_opt=None):
        from . import kernel as _kernel, mean as _mean
        from .model import GPParego
        rng = rng if rng is not None else np.random.default_rng()
        model = GPParego(-1, int(q), params, kernel=kernel if kernel is not None else _kernel.MaternFiveHalves,
                         mean=mean if mean is not None else _mean.Data, hp_opt=hp_opt, device=device, rng=rng)
        super().__init__(model, params, acqui, acqui_opt, rng)
        self._q = int(q)

    def optimize(self, sfun, dim_in: int, afun=_acqui.first_elem, reset: bool = True) -> None:
        if self._q == 1:
            super().optimize(sfun, dim_in, afun, reset)
            return
        if reset:
            self._samples, self._observations = [], []
            self._current_iteration = 0
        if self._total_iterations == 0 or reset:
            for _ in range(int(_get(self._params, "init_randomsampling", "samples"))):
                self.eval_and_add(sfun, self._rng.random(dim_in))
        if self._observations:
            self._model.compute(np.stack(self._samples), np.stack(self._observations))
        hp_period = int(get(self._params, "bayes_opt_boptimizer", "hp_period"))
        max_it = int(_get(self._params, "stop_maxiterations", "iterations"))
        propose = getattr(self._acqui_opt, "propose_batch", None)
        if propose is None:
            raise NotImplementedError("the acquisition optimiser proposes one point per call; q > 1 needs propose_batch")
        while self._current_iteration < max_it:
            acqui = self._acqui_cls(self._model, self._current_iteration, params=self._params)
            for x in distinct_rows(propose(acqui, dim_in, True)):
                if self._current_iteration >= max_it:
                    break
                self.eval_and_add(sfun, x)
                self._model.add_sample(self._samples[-1], self._observations[-1])
                if hp_period > 0 and (self._current_iteration + 1) % hp_period == 0:
                    self._model.optimize_hyperparams()
                self._current_iteration += 1
                self._total_iterations += 1
