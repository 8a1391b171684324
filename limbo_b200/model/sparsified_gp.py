"""limbo_b200.model.SparsifiedGP — drop-in mirror of limbo::model::SparsifiedGP (src/limbo/model/sparsified_gp.hpp:71-208).

A GP that keeps at most Params::model_sparse_gp::max_points samples: with more, it removes the densest samples first (the
smallest sum of the distances to the D nearest remaining samples) and fits the rest.  The sparsification runs on the device
(lb_sparsify, limbo_b200/csrc/sparsify.cu); the fit is the ordinary GP path."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _lib
from .. import kernel as _kernel
from .. import mean as _mean
from .. import params as _params
from .gp import GP


class SparsifiedGP(GP):
    def __init__(self, dim_in: int = -1, dim_out: int = -1, params=None, kernel=_kernel.MaternFiveHalves, mean=_mean.Data,
                 hp_opt=None, device: int = 0, precision: str = "fp64"):
        super().__init__(dim_in, dim_out, params=params, kernel=kernel, mean=mean, hp_opt=hp_opt, device=device, precision=precision)

    def max_points(self) -> int:
        return int(_params.get(self._params, "model_sparse_gp", "max_points"))

    def sparsify(self, samples):
        """Indices (ascending) of the samples _sparsify keeps (sparsified_gp.hpp:157-183)."""
        X = np.array(samples, dtype=np.float64, order="C")
        if X.ndim == 1:
            X = X[:, None]
        N, D = X.shape
        kept = np.empty(N, dtype=np.int64)
        n_kept = C.c_int64()
        _lib.check(self._lib.lb_sparsify(self._h, N, D, X.ctypes.data, self.max_points(), kept.ctypes.data, C.addressof(n_kept), None,
                                         None), "lb_sparsify")
        return kept[:n_kept.value]

    # ---- sparsified_gp.hpp:84-100 ----
    def compute(self, samples, observations, compute_kernel: bool = True) -> None:
        if len(samples) <= self.max_points():
            return super().compute(samples, observations, compute_kernel)
        X = np.array(samples, dtype=np.float64)
        Y = np.array(observations, dtype=np.float64)
        if X.ndim == 1:
            X = X[:, None]
        kept = self.sparsify(X)
        super().compute(X[kept], Y[kept], compute_kernel)

    # ---- sparsified_gp.hpp:104-118 ----
    def add_sample(self, sample, observation) -> None:
        if self.nb_samples() + 1 <= self.max_points():
            return super().add_sample(sample, observation)
        # past max_points the reference appends, then re-sparsifies the whole set and refits: the append is skipped here, the
        # result is the same
        sample = np.atleast_1d(np.asarray(sample, dtype=np.float64))
        observation = np.atleast_1d(np.asarray(observation, dtype=np.float64))
        if self.nb_samples() > 0:
            assert sample.size == self._dim_in and observation.size == self._dim_out
        X = np.vstack([self._sample_matrix(), sample[None, :]]) if self.nb_samples() else sample[None, :]
        Y = np.vstack([self._observations, observation[None, :]]) if self.nb_samples() else observation[None, :]
        self.compute(X, Y, True)
