"""limbo_b200.model.SPGP — drop-in mirror of limbo::experimental::model::SPGP (src/limbo/experimental/model/spgp.hpp:85-718),
Snelson and Ghahramani's sparse GP with M learned pseudo-inputs (FITC).  The likelihood, its gradient, the factorisation and the
prediction run on the device (lb_spgp_*, limbo_b200/csrc/spgp.cu); the hyper-parameter optimiser and the mean functor stay on the
host.  Single output, SE-ARD, as the reference's model is in practice.

Deliberate deviations (DESIGN.md §8):
  * the pseudo-inputs start from a permutation drawn from the model's numpy Generator (`rng`) instead of srand(time) /
    std::random_shuffle; the row-major write into the column-major xb block is kept;
  * the default optimiser is opt.Rprop (there is no NLopt here); any opt-style optimiser `f(fun, init, bounded)` is accepted;
  * at a non-positive pivot of Q or A the likelihood is (-inf, zero gradient), so optimisers step past the point."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from .. import _lib
from .. import kernel as _kernel
from .. import mean as _mean
from .. import opt as _opt
from .. import params as _params


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


class SPGP:
    def __init__(self, dim_in: int = -1, dim_out: int = -1, params=None, kernel=_kernel.SquaredExpARD, mean=_mean.Data,
                 hp_opt=None, device: int = 0, rng: np.random.Generator | None = None):
        self._params = params
        self._kernel_cls, self._mean_cls = kernel, mean
        self._dim_in, self._dim_out = dim_in, dim_out
        self._kernel_function = kernel(params, max(dim_in, 1))  # only the no-sample prior uses it (spgp.hpp:587-595)
        self._mean_function = mean(params, max(dim_out, 1))
        self._hp_optimize = hp_opt if hp_opt is not None else _opt.Rprop(params)
        self._rng = rng if rng is not None else np.random.default_rng()
        self._X = np.zeros((0, max(dim_in, 1)))
        self._observations = np.zeros((0, max(dim_out, 1)))
        self._obs_mean = np.zeros(max(dim_out, 1))
        self._m = 0
        self._w_init = None
        self._w = None
        self._optimized = False
        self._device = device
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.lb_spgp_create(C.byref(h), device), "lb_spgp_create")
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self._lib.lb_spgp_destroy(h)
            except Exception:
                pass
            self._h = None

    # ---- parameters (spgp.hpp:64-73) ----
    def _p(self, name: str):
        return _params.get(self._params, "model_spgp", name)

    def jitter(self) -> float:
        return float(self._p("jitter"))

    def _update_m(self) -> None:  # spgp.hpp:381-387
        m = int(float(self._p("samples_percent")) * self._X.shape[0] / 100)
        self._m = max(m, int(self._p("min_m")))

    # ---- data ----
    def _set(self, X, Y) -> None:  # _init (spgp.hpp:353-370)
        X = np.array(X, dtype=np.float64, order="C", copy=True)
        Y = np.array(Y, dtype=np.float64, copy=True)
        if X.ndim == 1:
            X = X[:, None]
        if Y.ndim == 1:
            Y = Y[:, None]
        assert X.shape[0] != 0 and X.shape[0] == Y.shape[0]
        if self._dim_in != X.shape[1]:
            self._dim_in = X.shape[1]
            self._kernel_function = self._kernel_cls(self._params, self._dim_in)
        if self._dim_out != Y.shape[1]:
            self._dim_out = Y.shape[1]
            self._mean_function = self._mean_cls(self._params, self._dim_out)
        self._X, self._observations = X, Y
        self._obs_mean = Y.mean(axis=0)
        # _compute_observations_zm (spgp.hpp:372-379): only the first output enters the model
        y_zm = np.ascontiguousarray(Y[:, 0] - self._mean_function.batch(X, self)[:, 0], dtype=np.float64)
        self._y_zm = y_zm
        self._update_m()
        _lib.check(self._lib.lb_spgp_set_data(self._h, X.shape[0], X.shape[1], _ptr(X), _ptr(y_zm)), "lb_spgp_set_data")

    def compute(self, samples, observations) -> None:  # spgp.hpp:132-152
        assert len(samples) != 0 and len(observations) != 0 and len(samples) == len(observations)
        self._set(samples, observations)
        self._optimize_init = True
        self._compute()

    def add_sample(self, sample, observation) -> None:  # spgp.hpp:155-186
        sample = np.atleast_1d(np.asarray(sample, dtype=np.float64))
        observation = np.atleast_1d(np.asarray(observation, dtype=np.float64))
        if self.nb_samples() == 0:
            X, Y = sample[None, :], observation[None, :]
        else:
            assert sample.size == self._dim_in and observation.size == self._dim_out
            X = np.vstack([self._X, sample[None, :]])
            Y = np.vstack([self._observations, observation[None, :]])
        self._set(X, Y)
        self._optimize_init = True
        self._compute()

    def recompute(self, update_obs_mean: bool = True) -> None:  # spgp.hpp:283-287
        self._optimize_init = True
        self._compute()

    def optimize_hyperparams(self) -> None:  # spgp.hpp:125-129
        self._optimize_init = True
        self._optimize_hyperparams()

    # ---- spgp.hpp:389-451 ----
    def initial_w(self) -> np.ndarray:
        """The reference's starting vector (spgp.hpp:414-426): pseudo-inputs are M distinct samples written ROW-major into the
        column-major xb block (kept as the reference has it), log b = -2 log((max - min) / 2), log c = log mean(y^2),
        log sig = log mean(y^2 / 4)."""
        X, y, M = self._X, self._y_zm, self._m
        N, D = X.shape
        perm = self._rng.permutation(N)
        w = np.empty((M + 1) * D + 2)
        for i in range(M):
            w[i * D:(i + 1) * D] = X[perm[i]]
        w[M * D:(M + 1) * D] = -2.0 * np.log((X.max(axis=0) - X.min(axis=0)) / 2.0)
        w[(M + 1) * D] = math.log(np.mean(y ** 2))
        w[(M + 1) * D + 1] = math.log(np.mean(y ** 2 / 4.0))
        return w

    def _optimize_hyperparams(self) -> None:
        if self._optimize_init or self._w_init is None:
            self._update_m()
            self._w_init = self.initial_w()
            self._optimize_init = False
        self._w = np.asarray(self._hp_optimize(lambda x, g: self._likelihood(x, g), self._w_init, False), dtype=np.float64)
        self._optimized = True

    def _compute(self, optimize: bool = True) -> None:
        if optimize:
            self._optimize_hyperparams()
        self.compute_at(self._w)

    def compute_at(self, w) -> None:
        """_compute(false) at HyperParams(w): the factors the queries use."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        _lib.check(self._lib.lb_spgp_compute(self._h, self._m, w.size, _ptr(w), self.jitter()), "lb_spgp_compute")
        self._w = w.copy()

    def _likelihood(self, w, eval_grad: bool = False):
        """_likelihood(w, eval_grad) (spgp.hpp:446-451): (-fw, -dfw); (-inf, 0) at a non-positive pivot."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        f = C.c_double()
        g = np.empty(w.size) if eval_grad else None
        rc = self._lib.lb_spgp_lik(self._h, self._m, w.size, _ptr(w), self.jitter(), C.addressof(f), _ptr(g) if g is not None else None)
        if rc > 0:
            return -math.inf, (np.zeros(w.size) if eval_grad else None)
        _lib.check(rc, "lb_spgp_lik")
        return f.value, g

    # ---- spgp.hpp:193-236, 582-610 ----
    def query_batch(self, Xq):
        """mu (Mq x 1) and sigma^2 (Mq) for Mq candidates in one device pass."""
        Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
        M = Xq.shape[0]
        P = max(self._dim_out, 1)
        if M == 0:
            return np.zeros((0, P)), np.zeros(0)
        mean = self._mean_function.batch(Xq, self)
        if self.nb_samples() == 0:
            return np.array(mean, dtype=np.float64), np.full(M, self._kernel_function.sigma_sq())
        mu = np.empty(M)
        s2 = np.empty(M)
        _lib.check(self._lib.lb_spgp_query(self._h, M, _ptr(Xq), int(self._optimized), _ptr(mu), _ptr(s2)), "lb_spgp_query")
        out = np.array(mean, dtype=np.float64)
        out[:, 0] += mu
        return out, s2

    def query(self, v):
        mu, s2 = self.query_batch(np.atleast_2d(np.asarray(v, dtype=np.float64)))
        return mu[0], float(s2[0])

    def predict(self, xt):
        return self.query_batch(xt)

    def mu(self, v) -> np.ndarray:
        return self.query(v)[0]

    def sigma(self, v) -> float:
        return self.query(v)[1]

    def acq_argmax_batch(self, acq_id: int, acq_params, Xq, return_values: bool = False):
        """Batched acquisition + argmax on the device (FirstElem aggregator).  Returns (best_value, best_index[, values])."""
        Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
        M = Xq.shape[0]
        ap = np.ascontiguousarray(np.atleast_1d(acq_params), dtype=np.float64)
        if ap.size < 2:
            ap = np.append(ap, 0.0)
        if self._mean_function.is_constant():
            mean0, mconst = None, float(np.asarray(self._mean_function(Xq[0], self))[0])
        else:
            mean0, mconst = np.ascontiguousarray(self._mean_function.batch(Xq, self)[:, 0]), 0.0
        vals = np.empty(M) if return_values else None
        best = C.c_double()
        idx = C.c_int64()
        _lib.check(self._lib.lb_spgp_acq_argmax(self._h, acq_id, _ptr(ap), M, _ptr(Xq), int(self._optimized),
                                                _ptr(mean0) if mean0 is not None else None, mconst,
                                                _ptr(vals) if vals is not None else None, C.addressof(best), C.addressof(idx)),
                   "lb_spgp_acq_argmax")
        if return_values:
            return best.value, idx.value, vals
        return best.value, idx.value

    def launch_count(self) -> int:
        return int(self._lib.lb_spgp_launch_count(self._h))

    # ---- accessors (spgp.hpp:238-293) ----
    def dim_in(self) -> int:
        assert self._dim_in != -1
        return self._dim_in

    def dim_out(self) -> int:
        assert self._dim_out != -1
        return self._dim_out

    def mean_function(self):
        return self._mean_function

    def kernel_function(self):
        return self._kernel_function

    def max_observation(self) -> np.ndarray:
        if self._observations.shape[1] > 1:
            print("WARNING max_observation with multi dimensional observations doesn't make sense")
        return np.array([self._observations.max()])

    def mean_observation(self) -> np.ndarray:
        return self._obs_mean if self.nb_samples() > 0 else np.zeros(max(self._dim_out, 1))

    def nb_samples(self) -> int:
        return self._X.shape[0]

    def nb_pseudo_samples(self) -> int:
        return 0 if self._w is None else self._m

    def samples(self):
        return list(self._X)

    def pseudo_samples(self):
        """The pseudo-inputs of HyperParams(w) (M x D, xb read column-major from w)."""
        if self._w is None:
            return []
        M, D = self._m, self._dim_in
        return list(self._w[:M * D].reshape(D, M).T.copy())

    def hyper_params(self) -> np.ndarray:
        return None if self._w is None else self._w.copy()
