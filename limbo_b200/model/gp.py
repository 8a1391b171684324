"""limbo_b200.model.GP — drop-in mirror of limbo::model::GP (src/limbo/model/gp.hpp:81-511)
whose numerical work runs on the GPU through the C ABI (include/limbo_b200.h).

Same member names, argument meaning and error behaviour as the reference's
template (asserts where the reference asserts).  Extensions that the
one-point-at-a-time reference lacks are suffixed ``_batch``.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from .. import _lib
from .. import kernel as _kernel
from .. import mean as _mean
from ._calls import acq_param_pair, argmax, candidates, cmaes, constant_mean, first_mean, first_mean_and_grad, ptr, values_and_grads


class GP:
    def __init__(self, dim_in: int = -1, dim_out: int = -1, params=None, kernel=_kernel.MaternFiveHalves,
                 mean=_mean.Data, hp_opt=None, device: int = 0, precision: str = "fp64"):
        # gp.hpp:84-88
        self._params = params
        self._kernel_cls, self._mean_cls = kernel, mean
        self._dim_in, self._dim_out = dim_in, dim_out
        self._kernel_function = kernel(params, dim_in) if dim_in > 0 else kernel(params, 1)
        self._mean_function = mean(params, dim_out) if dim_out > 0 else mean(params, 1)
        if hp_opt is None:
            from .hp_opt import NoLFOpt
            hp_opt = NoLFOpt(params)
        self._hp_optimize = hp_opt
        self._samples: list[np.ndarray] = []
        self._observations = np.zeros((0, max(dim_out, 1)))
        self._mean_vector = np.zeros((0, max(dim_out, 1)))
        self._obs_mean = np.zeros((0, max(dim_out, 1)))
        self._mean_observation = np.zeros(max(dim_out, 1))
        self._log_lik = 0.0
        self._log_loo_cv = 0.0
        self._inv_kernel_updated = False
        self._device = device
        self._lib = _lib.load()
        h = C.c_void_p()
        self._precision = {"fp64": 0, "tf32": 1, "fp16": 2, "fp16x3": 3}[precision]
        _lib.check(self._lib.lb_create(C.byref(h), device, self._precision), "lb_create")
        self._h = h
        self._host_cache: dict[str, np.ndarray] = {}

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self._lib.lb_destroy(h)
            except Exception:
                pass
            self._h = None

    # ---- copy semantics (kernel_lf_opt.hpp:79 copies the GP per evaluation) ----
    def copy(self) -> "GP":
        import copy as _copy
        g = type(self).__new__(type(self))
        g.__dict__.update({k: v for k, v in self.__dict__.items() if k not in ("_h", "_host_cache")})
        g._kernel_function = _copy.deepcopy(self._kernel_function)
        g._mean_function = _copy.deepcopy(self._mean_function)
        g._samples = list(self._samples)
        g._X = getattr(self, '_X', None)
        g._observations = self._observations.copy()
        g._mean_vector = self._mean_vector.copy()
        g._obs_mean = self._obs_mean.copy()
        g._mean_observation = self._mean_observation.copy()
        g._host_cache = {}
        h = C.c_void_p()
        _lib.check(self._lib.lb_clone(self._h, C.byref(h)), "lb_clone")
        g._h = h
        return g

    # ---- device plumbing ----
    def set_stream(self, stream_ptr: int | None) -> None:
        _lib.check(self._lib.lb_set_stream(self._h, C.c_void_p(stream_ptr or 0)), "lb_set_stream")
        self._stream_ptr = stream_ptr or 0

    def launch_count(self) -> int:
        return int(self._lib.lb_launch_count(self._h))

    def append_count(self) -> int:
        """how many add_sample calls took the incremental Cholesky path (lb_append) on this handle"""
        return int(self._lib.lb_debug_append_count(self._h))

    def _push_kernel(self) -> None:
        k = self._kernel_function
        own = np.ascontiguousarray(k.params(), dtype=np.float64)
        _lib.check(self._lib.lb_set_kernel(self._h, k.kernel_id, ptr(own), own.size, k.noise()), "lb_set_kernel")

    def _sample_matrix(self) -> np.ndarray:
        X = getattr(self, "_X", None)
        if X is None or X.shape[0] != len(self._samples):
            X = np.ascontiguousarray(np.stack(self._samples, axis=0), dtype=np.float64)
            self._X = X
        return X

    def _push_data(self) -> None:
        X = self._sample_matrix()
        Y = np.asfortranarray(self._obs_mean, dtype=np.float64)
        _lib.check(self._lib.lb_set_data(self._h, X.shape[0], X.shape[1], Y.shape[1], ptr(X), ptr(Y)), "lb_set_data")

    # ---- gp.hpp:88-116 ----
    def compute(self, samples, observations, compute_kernel: bool = True) -> None:
        assert len(samples) != 0
        assert len(observations) != 0
        assert len(samples) == len(observations)
        # std::vector<Eigen::VectorXd> in the reference; a 2-D array (one point per row) is taken as is
        # the reference copies the caller's vectors (gp.hpp:104-105: _samples = samples); never alias the caller's arrays
        X = np.array(samples, dtype=np.float64, order="C", copy=True)
        Y = np.array(observations, dtype=np.float64, order="C", copy=True)
        if X.ndim == 1:
            X = X[:, None]
        if Y.ndim == 1:
            Y = Y[:, None]
        if self._dim_in != X.shape[1]:
            self._dim_in = X.shape[1]
            self._kernel_function = self._kernel_cls(self._params, self._dim_in)
        if self._dim_out != Y.shape[1]:
            self._dim_out = Y.shape[1]
            self._mean_function = self._mean_cls(self._params, self._dim_out)
        self._samples = list(X)  # row views, no copies
        self._X = X
        self._observations = Y
        self._mean_observation = self._observations.mean(axis=0)
        self._compute_obs_mean()
        self._fitted = False
        if compute_kernel:
            self._compute_full_kernel()

    # ---- gp.hpp:119-122 ----
    def optimize_hyperparams(self) -> None:
        self._hp_optimize(self)

    # ---- gp.hpp:126-152 ----
    def add_sample(self, sample, observation) -> None:
        sample = np.atleast_1d(np.asarray(sample, dtype=np.float64))
        observation = np.atleast_1d(np.asarray(observation, dtype=np.float64))
        if len(self._samples) == 0:
            if self._dim_in != sample.size:
                self._dim_in = sample.size
                self._kernel_function = self._kernel_cls(self._params, self._dim_in)
            if self._dim_out != observation.size:
                self._dim_out = observation.size
                self._mean_function = self._mean_cls(self._params, self._dim_out)
            self._observations = np.zeros((0, self._dim_out))
        else:
            assert sample.size == self._dim_in
            assert observation.size == self._dim_out
        self._samples.append(sample)
        self._X = None
        self._observations = np.vstack([self._observations, observation[None, :]])
        self._mean_observation = self._observations.mean(axis=0)
        self._compute_obs_mean()
        self._compute_incremental_kernel()

    # ---- gp.hpp:159-191 ----
    def query(self, v):
        mu, s2 = self.query_batch(np.atleast_2d(np.asarray(v, dtype=np.float64)))
        return mu[0], float(s2[0])

    def mu(self, v) -> np.ndarray:
        return self.query(v)[0]

    def sigma(self, v) -> float:
        return self.query(v)[1]

    def query_batch(self, Xq):
        """mu (M x P) and sigma^2 (M) for M candidates in one device pass."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        P = max(self._dim_out, 1)
        if M == 0 or Xq.size == 0:
            return np.zeros((0, P)), np.zeros(0)
        self._push_prior_if_empty(Xq.shape[1])
        mu = np.empty((M, P))
        s2 = np.empty(M)
        _lib.check(self._lib.lb_query(self._h, M, ptr(Xq), ptr(mu), ptr(s2)), "lb_query")
        mu += self._mean_function.batch(Xq, self)  # gp.hpp:615
        return mu, s2

    def _push_prior_if_empty(self, d: int) -> None:
        # gp.hpp:161-163: without samples, mean(v) and k(v,v) + noise; the kernel state is still needed on the device
        if len(self._samples) != 0:
            return
        if self._dim_in != d:
            self._dim_in = d
            self._kernel_function = self._kernel_cls(self._params, d)
        if self._dim_out < 1:
            self._dim_out = 1
        _lib.check(self._lib.lb_set_data(self._h, 0, d, self._dim_out, None, None), "lb_set_data")
        self._push_kernel()

    def acq_argmax_batch(self, acq_id: int, acq_params, Xq, return_values: bool = False):
        """Fused batched acquisition + argmax on the device (FirstElem aggregator,
        bo_base.hpp:99-105).  Returns (best_value, best_index[, values])."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        ap = acq_param_pair(acq_params)
        mean0, mconst = first_mean(self, Xq)
        return argmax(self._lib, "lb_acq_argmax", M, return_values, self._h, acq_id, ptr(ap), M, ptr(Xq), ptr(mean0), mconst)

    def acq_argmax_cols(self, acq_id: int, acq_params, Xq, return_values: bool = False):
        """acq_argmax_batch in each of the P output columns from one query (lb_acq_argmax_cols): acq_params is P x 2 (row r: column r's
        alpha and 0, or f_max and jitter), and column r adds the mean's output r.  Returns (best_values (P), best_indices (P)[,
        values (M x P)])."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        P = max(self._dim_out, 1)
        ap = np.ascontiguousarray(np.asarray(acq_params, dtype=np.float64).reshape(P, 2))
        self._push_prior_if_empty(Xq.shape[1])
        mf = self._mean_function
        if mf.is_constant():
            mean, mconst = None, np.ascontiguousarray(np.asarray(mf(Xq[0], self), dtype=np.float64).reshape(P))
        else:
            mean, mconst = np.ascontiguousarray(np.asarray(mf.batch(Xq, self), dtype=np.float64).reshape(M, P)), np.zeros(P)
        vals = np.empty((M, P)) if return_values else None
        best, idx = np.empty(P), np.empty(P, dtype=np.int64)
        _lib.check(self._lib.lb_acq_argmax_cols(self._h, acq_id, P, ptr(ap), M, ptr(Xq), ptr(mean), ptr(mconst), ptr(vals), ptr(best),
                                                ptr(idx)), "lb_acq_argmax_cols")
        return (best, idx, vals) if return_values else (best, idx)

    def acq_cmaes_cols(self, acq_id: int, acq_params, starts, cols, lam: int = 0, sigma0: float = 0.5, generations: int = 100,
                       tolx: float = 1e-12, seed: int = 0, bounded: bool = True):
        """acq_cmaes_batch over the P columns of acq_argmax_cols (lb_acq_cmaes_cols): the instance started from starts[i] searches
        column cols[i], and every column needs one.  Returns (best_x (P x D), best_val (P), n_evals); NotImplementedError for a mean
        that depends on the input."""
        S = candidates(starts)
        D = S.shape[1]
        P = max(self._dim_out, 1)
        mf = self._mean_function
        if not mf.is_constant():
            raise NotImplementedError("the device CMA-ES takes input-free means only")
        self._push_prior_if_empty(D)
        mconst = np.ascontiguousarray(np.asarray(mf(np.zeros(D), self), dtype=np.float64).reshape(P))
        ap = np.ascontiguousarray(np.asarray(acq_params, dtype=np.float64).reshape(P, 2))
        c = np.ascontiguousarray(np.asarray(cols, dtype=np.int32).reshape(S.shape[0]))
        opts = _lib.CmaesOpts(int(lam), float(sigma0), int(generations), float(tolx), int(seed) & 0xFFFFFFFFFFFFFFFF, int(bool(bounded)))
        bx, bv, n = np.empty((P, D)), np.empty(P), C.c_int64()
        _lib.check(self._lib.lb_acq_cmaes_cols(self._h, acq_id, P, ptr(ap), ptr(mconst), C.byref(opts), S.shape[0], ptr(S), ptr(c), ptr(bx),
                                               ptr(bv), C.addressof(n)), "lb_acq_cmaes_cols")
        return bx, bv, n.value

    def eci_argmax_batch(self, constraint_model, f_max: float, jitter: float, Xq, return_values: bool = False):
        """Fused batched expected constrained improvement + argmax on the device (experimental/acqui/eci.hpp:76-130, FirstElem
        aggregator): this GP is the objective, `constraint_model` (a GP on the same device, or None for no constraints) gives
        Pf from its first output.  Returns (best_value, best_index[, values])."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        ep = np.array([f_max, jitter], dtype=np.float64)
        mean0, mconst = first_mean(self, Xq)
        con_h, cmean0, cconst = None, None, 0.0
        if constraint_model is not None:
            con_h = constraint_model._h
            if constraint_model.nb_samples() > 0:
                cmean0, cconst = first_mean(constraint_model, Xq)
        return argmax(self._lib, "lb_eci_argmax", M, return_values, self._h, con_h, ptr(ep), M, ptr(Xq), ptr(mean0), mconst, ptr(cmean0),
                      cconst)

    def ehvi_argmax_batch(self, other, ref_point, front, Xq, return_values: bool = False):
        """Fused batched two-objective expected hypervolume improvement + argmax on the device (experimental/acqui/ehvi.hpp:70-79,
        FirstElem aggregator): this GP models the first objective and `other` (a distinct GP on the same device) the second;
        front is the k x 2 array of current Pareto objective values, ref_point the reference point.  A model without samples
        scores with its prior.  Returns (best_value, best_index[, values])."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        F = np.ascontiguousarray(np.asarray(front, dtype=np.float64).reshape(-1, 2))
        r = np.ascontiguousarray(np.asarray(ref_point, dtype=np.float64).reshape(-1)[:2])
        for g in (self, other):
            g._push_prior_if_empty(Xq.shape[1])
        mean0, c0 = first_mean(self, Xq)
        mean1, c1 = first_mean(other, Xq)
        return argmax(self._lib, "lb_ehvi_argmax", M, return_values, self._h, other._h, ptr(r), F.shape[0], ptr(F) if F.size else None, M,
                      ptr(Xq), ptr(mean0), c0, ptr(mean1), c1)

    def ehvi3d_argmax_batch(self, m1, m2, ref_point, front, Xq, return_values: bool = False):
        """Fused batched three-objective expected hypervolume improvement + argmax on the device (ehvi3d_sliceupdate,
        src/ehvi/ehvi_sliceupdate.cc, FirstElem aggregator, each model's sigma() where a deviation is expected, as in
        ehvi_argmax_batch): this GP models the first objective, m1 and m2 (distinct GPs on the same device) the second and third;
        front is the k x 3 array of current Pareto objective values (k <= LB_EHVI3D_MAX_K = 256), ref_point the reference point
        (its first three entries are used).  A model without samples scores with its prior.  Returns (best_value,
        best_index[, values])."""
        Xq = candidates(Xq)
        M = Xq.shape[0]
        F = np.ascontiguousarray(np.asarray(front, dtype=np.float64).reshape(-1, 3))
        r = np.ascontiguousarray(np.asarray(ref_point, dtype=np.float64).reshape(-1)[:3])
        for g in (self, m1, m2):
            g._push_prior_if_empty(Xq.shape[1])
        means = [first_mean(g, Xq) for g in (self, m1, m2)]
        return argmax(self._lib, "lb_ehvi3d_argmax", M, return_values, self._h, m1._h, m2._h, ptr(r), F.shape[0], ptr(F) if F.size else None,
                      M, ptr(Xq), *[a for m, c in means for a in (ptr(m), c)])

    def acq_cmaes_batch(self, acq_id: int, acq_params, starts, **opts):
        """Batched CMA-ES on the device (lb_acq_cmaes) over UCB / GP_UCB (acq_id 0) or EI (acq_id 1), parameters as
        acq_argmax_batch: one instance from each row of `starts` (R x D).  opts: lam (0: 4 + floor(3 ln D)), sigma0, generations,
        tolx, seed, bounded.  Returns (best_x, best_val, n_evals); NotImplementedError for a mean that depends on the input."""
        S = candidates(starts)
        mconst = constant_mean(self, S.shape[1])
        self._push_prior_if_empty(S.shape[1])
        return cmaes(self._lib, "lb_acq_cmaes", S.shape[1], self._h, acq_id, ptr(acq_param_pair(acq_params)), mconst, S, **opts)

    def ehvi_cmaes_batch(self, others, ref_point, front, starts, **opts):
        """Batched CMA-ES on the device (lb_ehvi_cmaes) over the two-objective (others = [m1]) or three-objective (others = [m1,
        m2]) EHVI of ehvi_argmax_batch / ehvi3d_argmax_batch; starts and opts as acq_cmaes_batch.  Returns (best_x, best_val,
        n_evals); NotImplementedError for a mean that depends on the input."""
        S = candidates(starts)
        D = S.shape[1]
        models = [self, *others]
        K = len(models)
        assert K in (2, 3)
        F = np.ascontiguousarray(np.asarray(front, dtype=np.float64).reshape(-1, K))
        r = np.ascontiguousarray(np.asarray(ref_point, dtype=np.float64).reshape(-1)[:K])
        consts = [constant_mean(g, D) for g in models] + [0.0] * (3 - K)
        for g in models:
            g._push_prior_if_empty(D)
        return cmaes(self._lib, "lb_ehvi_cmaes", D, self._h, models[1]._h, models[2]._h if K == 3 else None, ptr(r), F.shape[0],
                     ptr(F) if F.size else None, *consts, S, **opts)

    def eci_cmaes_batch(self, constraint_model, f_max: float, jitter: float, starts, **opts):
        """Batched CMA-ES on the device (lb_eci_cmaes) over the expected constrained improvement of eci_argmax_batch: this GP is the
        objective, `constraint_model` a GP on the same device or None (a constraint without samples gives Pf = 1, as None does);
        starts and opts as acq_cmaes_batch.  Without objective samples every value is 0: (the first start, 0.0, 0).  Returns
        (best_x, best_val, n_evals); NotImplementedError for a mean of either model that depends on the input."""
        S = candidates(starts)
        D = S.shape[1]
        mconst = constant_mean(self, D)
        con_h, cconst = None, 0.0
        if constraint_model is not None:
            con_h = constraint_model._h
            cconst = constant_mean(constraint_model, D)
            if constraint_model.nb_samples() == 0:
                cconst = 0.0
        self._push_prior_if_empty(D)  # the search needs the input dimension even when it scores nothing
        return cmaes(self._lib, "lb_eci_cmaes", D, self._h, con_h, ptr(np.array([f_max, jitter], dtype=np.float64)), mconst, cconst, S,
                     **opts)

    def query_grad_batch(self, Xq):
        """mu (M x P), sigma^2 (M) and their gradients with respect to the candidates, grad mu (M x D, of the first output) and
        grad sigma^2 (M x D), in one device pass (lb_query_grad); the mean's value and input gradient are added.  Raises
        NotImplementedError for a mean without an input gradient (mean.BaseMean.grad_x)."""
        Xq = candidates(Xq)
        M, D = Xq.shape
        P = max(self._dim_out, 1)
        mgrad = self._mean_function.grad_x(Xq, self)
        self._push_prior_if_empty(D)
        mu, s2 = np.empty((M, P)), np.empty(M)
        dmu, ds2 = np.empty((M, D)), np.empty((M, D))
        _lib.check(self._lib.lb_query_grad(self._h, M, ptr(Xq), ptr(mu), ptr(s2), ptr(dmu), ptr(ds2)), "lb_query_grad")
        mu += self._mean_function.batch(Xq, self)
        dmu += mgrad[:, 0, :]
        return mu, s2, dmu, ds2

    def acq_grad_batch(self, acq_id: int, acq_params, Xq):
        """Acquisition values (M) and gradients (M x D) of UCB / GP_UCB (acq_id 0) or EI (acq_id 1) with the FirstElem aggregator,
        in one device pass (lb_acq_grad); parameters and values as acq_argmax_batch."""
        Xq = candidates(Xq)
        M, D = Xq.shape
        ap = acq_param_pair(acq_params)
        mean0, mconst, mgrad = first_mean_and_grad(self, Xq, self._push_prior_if_empty)
        return values_and_grads(self._lib, "lb_acq_grad", M, D, self._h, acq_id, ptr(ap), M, ptr(Xq), ptr(mean0), mconst, ptr(mgrad))

    def eci_grad_batch(self, constraint_model, f_max: float, jitter: float, Xq):
        """ECI values (M) and gradients (M x D) with respect to the candidates, in one device pass over both models (lb_eci_grad);
        arguments and values as eci_argmax_batch.  The means' input gradients are added; NotImplementedError for a mean without one."""
        Xq = candidates(Xq)
        M, D = Xq.shape
        ep = np.array([f_max, jitter], dtype=np.float64)
        mean0, mconst, mgrad = first_mean_and_grad(self, Xq, self._push_prior_if_empty)
        con_h, cmean0, cconst, cgrad = None, None, 0.0, None
        if constraint_model is not None:
            con_h = constraint_model._h
            if constraint_model.nb_samples() > 0:
                cmean0, cconst, cgrad = first_mean_and_grad(constraint_model, Xq)
        return values_and_grads(self._lib, "lb_eci_grad", M, D, self._h, con_h, ptr(ep), M, ptr(Xq), ptr(mean0), mconst, ptr(mgrad),
                                ptr(cmean0), cconst, ptr(cgrad))

    def ehvi_grad_batch(self, other, ref_point, front, Xq):
        """Two-objective EHVI values (M) and gradients (M x D) with respect to the candidates, in one device pass over both models
        (lb_ehvi_grad); arguments and values as ehvi_argmax_batch.  The means' input gradients are added; NotImplementedError for a
        mean without one."""
        Xq = candidates(Xq)
        M, D = Xq.shape
        F = np.ascontiguousarray(np.asarray(front, dtype=np.float64).reshape(-1, 2))
        r = np.ascontiguousarray(np.asarray(ref_point, dtype=np.float64).reshape(-1)[:2])
        mean0, c0, g0 = first_mean_and_grad(self, Xq, self._push_prior_if_empty)
        mean1, c1, g1 = first_mean_and_grad(other, Xq, other._push_prior_if_empty)
        return values_and_grads(self._lib, "lb_ehvi_grad", M, D, self._h, other._h, ptr(r), F.shape[0], ptr(F) if F.size else None, M,
                                ptr(Xq), ptr(mean0), c0, ptr(g0), ptr(mean1), c1, ptr(g1))

    # ---- accessors gp.hpp:194-238 ----
    def dim_in(self) -> int:
        assert self._dim_in != -1
        return self._dim_in

    def dim_out(self) -> int:
        assert self._dim_out != -1
        return self._dim_out

    def kernel_function(self):
        return self._kernel_function

    def mean_function(self):
        return self._mean_function

    def max_observation(self) -> np.ndarray:
        if self._observations.shape[1] > 1:
            print("WARNING max_observation with multi dimensional observations doesn't make sense")
        return np.array([self._observations.max()])

    def mean_observation(self) -> np.ndarray:
        assert self._dim_out > 0
        return self._mean_observation if len(self._samples) > 0 else np.zeros(self._dim_out)

    def mean_vector(self) -> np.ndarray:
        return self._mean_vector

    def obs_mean(self) -> np.ndarray:
        return self._obs_mean

    def nb_samples(self) -> int:
        return len(self._samples)

    # ---- gp.hpp:241-252 ----
    def recompute(self, update_obs_mean: bool = True, update_full_kernel: bool = True) -> None:
        assert len(self._samples) != 0
        if update_obs_mean:
            self._compute_obs_mean()
        if update_full_kernel:
            self._compute_full_kernel()
        else:
            self._compute_alpha()

    # ---- gp.hpp:254-264 ----
    def compute_inv_kernel(self) -> None:
        _lib.check(self._lib.lb_compute_inv_kernel(self._h), "lb_compute_inv_kernel")
        self._inv_kernel_updated = True

    # ---- gp.hpp:267-282 ----
    def compute_log_lik(self) -> float:
        out = C.c_double()
        _lib.check(self._lib.lb_log_lik(self._h, C.addressof(out)), "lb_log_lik")
        self._log_lik = out.value
        return self._log_lik

    # ---- gp.hpp:285-311 ----
    def compute_kernel_grad_log_lik(self) -> np.ndarray:
        k = self._kernel_function
        g = np.empty(k.h_params_size())
        _lib.check(self._lib.lb_kernel_grad_log_lik(self._h, int(k.optimize_noise()), ptr(g)), "lb_kernel_grad_log_lik")
        self._inv_kernel_updated = True
        return g

    # ---- gp.hpp:267-311 at R kernel states in one call (lb_lml_grad_batch); the model is not changed ----
    def lml_grad_batch(self, H, compute_grad: bool = True):
        """compute_log_lik and compute_kernel_grad_log_lik as a copy of this GP would return them after
        kernel_function().set_h_params(H[r]) and recompute(False), for every row r of H (R x h_params_size(), the noise
        entry last when optimize_noise: noise = exp(2 p), kernel.hpp).  Returns (lik (R,), grad (R x h_params_size()) or None,
        info (R,)): info[r] > 0 is the 1-based first non-positive pivot of that row's factor, where lik and grad are NaN."""
        k = self._kernel_function
        H = np.ascontiguousarray(np.atleast_2d(np.asarray(H, dtype=np.float64)))
        R, nh = H.shape
        assert nh == k.h_params_size()
        nk = k.params_size()
        own = np.ascontiguousarray(H[:, :nk])
        if k.optimize_noise():  # kernel.hpp:116-123, the same exp the kernel functor takes
            noise = np.array([math.exp(2.0 * float(p)) for p in H[:, nk]], dtype=np.float64)
        else:
            noise = np.full(R, k.noise(), dtype=np.float64)
        lik = np.empty(R)
        grad = np.empty((R, nh)) if compute_grad else None
        info = np.empty(R, dtype=np.int32)
        _lib.check(self._lib.lb_lml_grad_batch(self._h, k.kernel_id, R, nk, ptr(own), ptr(noise), int(k.optimize_noise()), ptr(lik),
                                               ptr(grad), ptr(info)), "lb_lml_grad_batch")
        return lik, grad, info

    # ---- gp.hpp:313-330: obs_mean^T K^-1 on the device (lb_kinv_obs_mean); the mean functor's gradient is host code ----
    def compute_mean_grad_log_lik(self) -> np.ndarray:
        n = self.nb_samples()
        w = np.empty((n, self._dim_out), order="F")
        _lib.check(self._lib.lb_kinv_obs_mean(self._h, ptr(w)), "lb_kinv_obs_mean")
        self._inv_kernel_updated = True
        grad = np.zeros(self._mean_function.h_params_size())
        for n_obs in range(n):
            mg = np.asarray(self._mean_function.grad(self._samples[n_obs], self), dtype=np.float64)
            for i_obs in range(self._dim_out):
                grad += w[n_obs, i_obs] * mg[i_obs]
        return grad

    # ---- gp.hpp:339-351 ----
    def compute_log_loo_cv(self) -> float:
        out = C.c_double()
        _lib.check(self._lib.lb_log_loo_cv(self._h, C.addressof(out)), "lb_log_loo_cv")
        self._inv_kernel_updated = True
        self._log_loo_cv = out.value
        return self._log_loo_cv

    # ---- gp.hpp:353-399 ----
    def compute_kernel_grad_log_loo_cv(self) -> np.ndarray:
        k = self._kernel_function
        g = np.empty(k.h_params_size())
        _lib.check(self._lib.lb_kernel_grad_log_loo_cv(self._h, int(k.optimize_noise()), ptr(g)), "lb_kernel_grad_log_loo_cv")
        self._inv_kernel_updated = True
        return g

    def get_log_loo_cv(self) -> float:
        return self._log_loo_cv

    def set_log_loo_cv(self, v: float) -> None:
        self._log_loo_cv = v

    def get_log_lik(self) -> float:
        return self._log_lik

    def set_log_lik(self, v: float) -> None:
        self._log_lik = v

    # ---- gp.hpp:404-436 ----
    def _get(self, what: int, shape) -> np.ndarray:
        out = np.empty(shape, order="F")
        _lib.check(self._lib.lb_get(self._h, what, ptr(out)), "lb_get")
        return out

    def matrixL(self) -> np.ndarray:
        n = self.nb_samples()
        return self._get(_lib.GET_L, (n, n))

    def alpha(self) -> np.ndarray:
        return self._get(_lib.GET_ALPHA, (self.nb_samples(), self._dim_out))

    def kernel_matrix(self) -> np.ndarray:
        n = self.nb_samples()
        return self._get(_lib.GET_K, (n, n))

    def inv_kernel(self) -> np.ndarray:
        n = self.nb_samples()
        self._inv_kernel_updated = True
        return self._get(_lib.GET_KINV, (n, n))

    def samples(self):
        return self._samples

    def observations(self):
        return [self._observations[i] for i in range(self._observations.shape[0])]

    def observations_matrix(self) -> np.ndarray:
        return self._observations

    def inv_kernel_computed(self) -> bool:
        return self._inv_kernel_updated

    # ---- gp.hpp:439-511 save / load ----
    def save(self, archive) -> None:
        from ..serialize import TextArchive
        if isinstance(archive, str):
            archive = TextArchive(archive)
        if self._kernel_function.h_params_size() > 0:
            archive.save(self._kernel_function.h_params(), "kernel_params")
        if self._mean_function.h_params_size() > 0:
            archive.save(self._mean_function.h_params(), "mean_params")
        archive.save(self._samples, "samples")
        archive.save(self._observations, "observations")
        archive.save(self.matrixL(), "matrixL")
        archive.save(self.alpha(), "alpha")

    def load(self, archive, recompute: bool = True) -> None:
        from ..serialize import TextArchive
        if isinstance(archive, str):
            archive = TextArchive(archive)
        self._samples = archive.load_vector_list("samples")
        self._X = None
        self._observations = archive.load_matrix("observations")
        self._dim_in = self._samples[0].size
        self._kernel_function = self._kernel_cls(self._params, self._dim_in)
        if self._kernel_function.h_params_size() > 0:
            hp = archive.load_vector("kernel_params")
            assert hp.size == self._kernel_function.h_params_size()
            self._kernel_function.set_h_params(hp)
        self._dim_out = self._observations.shape[1]
        self._mean_function = self._mean_cls(self._params, self._dim_out)
        if self._mean_function.h_params_size() > 0:
            hp = archive.load_vector("mean_params")
            assert hp.size == self._mean_function.h_params_size()
            self._mean_function.set_h_params(hp)
        self._mean_observation = self._observations.mean(axis=0)
        if recompute:
            self.recompute(True, True)
        else:  # gp.hpp:505-509: adopt the stored factor and alpha
            self._compute_obs_mean()
            self._push_data()
            self._push_kernel()
            L = np.asfortranarray(archive.load_matrix("matrixL"))
            A = np.asfortranarray(archive.load_matrix("alpha").reshape(len(self._samples), self._dim_out))
            _lib.check(self._lib.lb_load_factor(self._h, ptr(L), ptr(A)), "lb_load_factor")
            self._inv_kernel_updated = False

    # ---- protected helpers (same names as the reference) ----
    def _compute_obs_mean(self) -> None:  # gp.hpp:537-548
        assert len(self._samples) != 0
        X = self._sample_matrix()
        assert X.shape[1] == self._dim_in
        self._mean_vector = np.asarray(self._mean_function.batch(X, self), dtype=np.float64).reshape(len(self._samples), self._dim_out)
        self._obs_mean = self._observations - self._mean_vector

    def _compute_full_kernel(self) -> None:  # gp.hpp:550-571
        self._push_data()
        self._push_kernel()
        rc = self._lib.lb_fit(self._h)
        self._chol_info = rc
        if rc < 0:
            _lib.check(rc, "lb_fit")
        # rc > 0: non positive-definite K.  The reference never checks Eigen's info() (gp.hpp:565):
        # NaNs propagate.  We keep that behaviour but remember the pivot (chol_info()).
        self._inv_kernel_updated = False

    def chol_info(self) -> int:
        return getattr(self, "_chol_info", 0)

    def _compute_incremental_kernel(self) -> None:  # gp.hpp:573-603
        n = len(self._samples)
        if n == 1 or int(self._lib.lb_nb_samples(self._h)) != n - 1:
            self._compute_full_kernel()
            return
        self._push_kernel()  # unchanged functor state keeps the factor (lb_set_kernel compares)
        x = np.ascontiguousarray(self._samples[-1])
        Y = np.asfortranarray(self._obs_mean)
        rc = self._lib.lb_append(self._h, ptr(x), ptr(Y))
        if rc == -3:  # factor not resident (compute(..., compute_kernel=False) before, or the h-params changed since the fit)
            self._compute_full_kernel()
            return
        if rc < 0:
            _lib.check(rc, "lb_append")
        self._chol_info = rc
        self._inv_kernel_updated = False

    def _compute_alpha(self) -> None:  # gp.hpp:605-611
        Y = np.asfortranarray(self._obs_mean)
        rc = self._lib.lb_refit_alpha(self._h, ptr(Y))
        if rc < 0:
            _lib.check(rc, "lb_refit_alpha")


def GPBasic(params=None, **kw) -> GP:
    """gp.hpp:636-637"""
    from .hp_opt import NoLFOpt
    return GP(params=params, kernel=_kernel.MaternFiveHalves, mean=_mean.Data, hp_opt=NoLFOpt(params), **kw)


def GPOpt(params=None, **kw) -> GP:
    """gp.hpp:641-642"""
    from .hp_opt import KernelLFOpt
    return GP(params=params, kernel=_kernel.SquaredExpARD, mean=_mean.Data, hp_opt=KernelLFOpt(params), **kw)
