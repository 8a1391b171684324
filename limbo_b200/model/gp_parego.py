"""limbo_b200.model.GPParego — ParEGO's scalarised model (experimental/model/gp_parego.hpp:76-118) over model.GP, with q weight
vectors at once (qParEGO, Daulton et al., 2020): a GP with q output columns built over K-objective data, column r holding the
augmented Tchebycheff scalarisation of the raw observations under its own weight vector lambda_r.  All q columns share the
samples, hence one factor and one query; they differ only in alpha.  DESIGN.md §4.16."""
from __future__ import annotations

import numpy as np

from .. import kernel as _kernel
from .. import mean as _mean
from ..params import get
from .gp import GP


def normalise(draw) -> np.ndarray:
    """lambda / lambda.sum() (gp_parego.hpp:105-107) of one raw draw, the sum taken in sequence from 0 as the reference's Eigen
    stand-in does"""
    draw = np.asarray(draw, dtype=np.float64)
    s = 0.0
    for v in draw:
        s += float(v)
    return draw / s


def scalarise(lam, F, rho: float) -> np.ndarray:
    """gp_parego.hpp:108-115 for one normalised weight vector lam (K) over the N x K observations F: y = max(lam * f) + rho *
    sum(lam * f), the max first, then the sum in sequence from 0, then y + rho * s (two roundings, no fused multiply-add)"""
    P = np.asarray(F, dtype=np.float64) * np.asarray(lam, dtype=np.float64)[None, :]
    y = P.max(axis=1)
    s = np.zeros(P.shape[0])
    for k in range(P.shape[1]):
        s = s + P[:, k]
    return y + rho * s


class GPParego(GP):
    """A GP with q = dim_out scalarised columns over K-objective observations.  compute() and add_sample() take the raw K-objective
    observations, keep them (raw_observations()), draw q new weight vectors from the model's numpy Generator (one rng.random(K)
    each, normalised by its sum) and rescalarise every sample; add_sample() then extends the factor by one row and re-solves alpha
    against the rescalarised columns (lb_append) instead of refactorising, as the reference's compute() would.  `lambdas` (q x K raw
    draws, normalised here) replaces the draw of one call, so that tests can pin it.  mean::Data and every other mean apply per
    column; max_observation() and obs_mean() are those of the scalarised columns."""

    def __init__(self, dim_in: int = -1, dim_out: int = 1, params=None, kernel=_kernel.MaternFiveHalves, mean=_mean.Data, hp_opt=None,
                 device: int = 0, precision: str = "fp64", rng: np.random.Generator | None = None):
        assert dim_out >= 1
        if precision != "fp64":
            raise NotImplementedError("ParEGO runs on fp64 handles only")
        super().__init__(dim_in, dim_out, params, kernel, mean, hp_opt, device, precision)
        self._q = dim_out
        self._rng = rng if rng is not None else np.random.default_rng()
        self._raw = np.zeros((0, 0))
        self._lambda = np.zeros((dim_out, 0))
        self._draws = 0

    def nb_columns(self) -> int:
        return self._q

    def nb_objs(self) -> int:
        return self._raw.shape[1]

    def raw_observations(self) -> np.ndarray:
        return self._raw

    def lambdas(self) -> np.ndarray:
        """the q x K normalised weight vectors of the last compute / add_sample"""
        return self._lambda

    def lambda_draws(self) -> int:
        """weight vectors drawn so far (q per compute / add_sample)"""
        return self._draws

    def _rho(self) -> float:
        return float(get(self._params, "model_gp_parego", "rho"))

    def _scalarised(self, lambdas) -> np.ndarray:
        K = self._raw.shape[1]
        if lambdas is None:
            draws = [self._rng.random(K) for _ in range(self._q)]
        else:
            draws = np.asarray(lambdas, dtype=np.float64).reshape(self._q, K)
        self._lambda = np.stack([normalise(d) for d in draws])
        self._draws += self._q
        return np.stack([scalarise(lam, self._raw, self._rho()) for lam in self._lambda], axis=1)

    def compute(self, samples, observations, compute_kernel: bool = True, lambdas=None) -> None:  # gp_parego.hpp:83-90
        raw = np.array(observations, dtype=np.float64, order="C", copy=True)
        self._raw = raw[:, None] if raw.ndim == 1 else raw
        super().compute(samples, self._scalarised(lambdas), compute_kernel)

    def add_sample(self, sample, observation, lambdas=None) -> None:  # gp_parego.hpp:92-98, incremental
        observation = np.atleast_1d(np.asarray(observation, dtype=np.float64))
        sample = np.atleast_1d(np.asarray(sample, dtype=np.float64))
        if len(self._samples) == 0:
            self.compute(sample[None, :], observation[None, :], lambdas=lambdas)
            return
        assert sample.size == self._dim_in and observation.size == self._raw.shape[1]
        self._raw = np.vstack([self._raw, observation[None, :]])
        self._samples.append(sample)
        self._X = None
        self._observations = self._scalarised(lambdas)
        self._mean_observation = self._observations.mean(axis=0)
        self._compute_obs_mean()
        self._compute_incremental_kernel()

    def max_observation(self) -> np.ndarray:
        return self._observations.max(axis=0)
