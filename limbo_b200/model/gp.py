"""limbo_b200.model.GP — drop-in mirror of limbo::model::GP (src/limbo/model/gp.hpp:81-511)
whose numerical work runs on the GPU through the C ABI (include/limbo_b200.h).

Same member names, argument meaning and error behaviour as the reference's
template (asserts where the reference asserts).  Extensions that the
one-point-at-a-time reference lacks are suffixed ``_batch``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _lib
from .. import kernel as _kernel
from .. import mean as _mean


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


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
        _lib.check(self._lib.lb_set_kernel(self._h, k.kernel_id, _ptr(own), own.size, k.noise()), "lb_set_kernel")

    def _sample_matrix(self) -> np.ndarray:
        X = getattr(self, "_X", None)
        if X is None or X.shape[0] != len(self._samples):
            X = np.ascontiguousarray(np.stack(self._samples, axis=0), dtype=np.float64)
            self._X = X
        return X

    def _push_data(self) -> None:
        X = self._sample_matrix()
        Y = np.asfortranarray(self._obs_mean, dtype=np.float64)
        _lib.check(self._lib.lb_set_data(self._h, X.shape[0], X.shape[1], Y.shape[1], _ptr(X), _ptr(Y)), "lb_set_data")

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
        Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
        M = Xq.shape[0]
        P = max(self._dim_out, 1)
        if M == 0 or Xq.size == 0:
            return np.zeros((0, P)), np.zeros(0)
        if len(self._samples) == 0:
            # gp.hpp:161-163: mean(v) and k(v,v) + noise; the kernel state is still needed on the device
            self._ensure_dims_for_prior(Xq.shape[1])
        mu = np.empty((M, P))
        s2 = np.empty(M)
        _lib.check(self._lib.lb_query(self._h, M, _ptr(Xq), _ptr(mu), _ptr(s2)), "lb_query")
        mu += self._mean_function.batch(Xq, self)  # gp.hpp:615
        return mu, s2

    def _ensure_dims_for_prior(self, d: int) -> None:
        if self._dim_in != d:
            self._dim_in = d
            self._kernel_function = self._kernel_cls(self._params, d)
        if self._dim_out < 1:
            self._dim_out = 1
        X = np.zeros((0, d))
        Y = np.zeros((0, self._dim_out))
        _lib.check(self._lib.lb_set_data(self._h, 0, d, self._dim_out, None, None), "lb_set_data")
        self._push_kernel()

    def acq_argmax_batch(self, acq_id: int, acq_params, Xq, return_values: bool = False):
        """Fused batched acquisition + argmax on the device (FirstElem aggregator,
        bo_base.hpp:99-105).  Returns (best_value, best_index[, values])."""
        Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
        M = Xq.shape[0]
        ap = np.ascontiguousarray(np.atleast_1d(acq_params), dtype=np.float64)
        if ap.size < 2:
            ap = np.append(ap, 0.0)
        mean0, mconst = self._first_mean(Xq)
        mptr = _ptr(mean0) if mean0 is not None else None
        vals = np.empty(M) if return_values else None
        best = C.c_double()
        idx = C.c_int64()
        _lib.check(self._lib.lb_acq_argmax(self._h, acq_id, _ptr(ap), M, _ptr(Xq), mptr, mconst,
                                           _ptr(vals) if vals is not None else None, C.addressof(best), C.addressof(idx)),
                   "lb_acq_argmax")
        if return_values:
            return best.value, idx.value, vals
        return best.value, idx.value

    def eci_argmax_batch(self, constraint_model, f_max: float, jitter: float, Xq, return_values: bool = False):
        """Fused batched expected constrained improvement + argmax on the device (experimental/acqui/eci.hpp:76-130, FirstElem
        aggregator): this GP is the objective, `constraint_model` (a GP on the same device, or None for no constraints) gives
        Pf from its first output.  Returns (best_value, best_index[, values])."""
        Xq = np.ascontiguousarray(np.atleast_2d(Xq), dtype=np.float64)
        M = Xq.shape[0]
        ep = np.array([f_max, jitter], dtype=np.float64)
        mean0, mconst = self._first_mean(Xq)
        con_h, cmean0, cconst = None, None, 0.0
        if constraint_model is not None:
            con_h = constraint_model._h
            if constraint_model.nb_samples() > 0:
                cmean0, cconst = constraint_model._first_mean(Xq)
        vals = np.empty(M) if return_values else None
        best = C.c_double()
        idx = C.c_int64()
        _lib.check(self._lib.lb_eci_argmax(self._h, con_h, _ptr(ep), M, _ptr(Xq), _ptr(mean0) if mean0 is not None else None, mconst,
                                           _ptr(cmean0) if cmean0 is not None else None, cconst,
                                           _ptr(vals) if vals is not None else None, C.addressof(best), C.addressof(idx)),
                   "lb_eci_argmax")
        if return_values:
            return best.value, idx.value, vals
        return best.value, idx.value

    def _first_mean(self, Xq):
        """First output of the mean functor at every candidate, as (array, 0.0), or (None, constant) for a constant mean."""
        if self._mean_function.is_constant():
            return None, float(np.asarray(self._mean_function(Xq[0], self))[0])
        return np.ascontiguousarray(self._mean_function.batch(Xq, self)[:, 0]), 0.0

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
        _lib.check(self._lib.lb_kernel_grad_log_lik(self._h, int(k.optimize_noise()), _ptr(g)), "lb_kernel_grad_log_lik")
        self._inv_kernel_updated = True
        return g

    # ---- gp.hpp:313-330: obs_mean^T K^-1 on the device (lb_kinv_obs_mean); the mean functor's gradient is host code ----
    def compute_mean_grad_log_lik(self) -> np.ndarray:
        n = self.nb_samples()
        w = np.empty((n, self._dim_out), order="F")
        _lib.check(self._lib.lb_kinv_obs_mean(self._h, _ptr(w)), "lb_kinv_obs_mean")
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
        _lib.check(self._lib.lb_kernel_grad_log_loo_cv(self._h, int(k.optimize_noise()), _ptr(g)), "lb_kernel_grad_log_loo_cv")
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
        _lib.check(self._lib.lb_get(self._h, what, _ptr(out)), "lb_get")
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
            _lib.check(self._lib.lb_load_factor(self._h, _ptr(L), _ptr(A)), "lb_load_factor")
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
        rc = self._lib.lb_append(self._h, _ptr(x), _ptr(Y))
        if rc == -3:  # factor not resident (compute(..., compute_kernel=False) before, or the h-params changed since the fit)
            self._compute_full_kernel()
            return
        if rc < 0:
            _lib.check(rc, "lb_append")
        self._chol_info = rc
        self._inv_kernel_updated = False

    def _compute_alpha(self) -> None:  # gp.hpp:605-611
        Y = np.asfortranarray(self._obs_mean)
        rc = self._lib.lb_refit_alpha(self._h, _ptr(Y))
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
