"""Restatement of ParEGO's model (experimental/model/gp_parego.hpp:76-118) over the oracle GP (oracle.OracleGP), with q weight
vectors at once: the augmented Tchebycheff scalarisation (normalise, scalarise; written apart from limbo_b200.model.gp_parego's), mean::Data
per column, a full fit on compute and the incremental update (OracleGP.append with every row rescalarised) on add_sample.  The weight
vectors are always given (raw draws, q x K): the reference's come from an auto-seeded generator and cannot be replayed."""
from __future__ import annotations

import numpy as np

from . import oracle as O


def normalise(draw) -> np.ndarray:
    """gp_parego.hpp:105-107, element by element: lambda / sum(lambda), the sum in sequence from 0"""
    total = 0.0
    for v in draw:
        total += float(v)
    return np.array([float(v) / total for v in draw])


def scalarise(lam, F, rho: float) -> np.ndarray:
    """gp_parego.hpp:108-115, one observation at a time in Python floats: y = max_k lam_k f_k, s = sum_k lam_k f_k (in sequence
    from 0), y + rho s"""
    out = []
    for f in np.asarray(F, dtype=np.float64):
        p = [float(l) * float(v) for l, v in zip(lam, f)]
        s = 0.0
        for v in p:
            s += v
        out.append(max(p) + rho * s)
    return np.array(out)


class OracleParego:
    """q scalarised columns over K-objective observations, kernel (kernel_id, hparams, noise) fixed, mean::Data"""

    def __init__(self, kernel_id: int, hparams, noise: float, rho: float = 0.05):
        self.kernel_id, self.hparams, self.noise, self.rho = kernel_id, np.asarray(hparams, dtype=np.float64), float(noise), float(rho)
        self.gp = O.OracleGP()
        self.X = np.zeros((0, 0))
        self.F = np.zeros((0, 0))

    def _columns(self, draws) -> np.ndarray:
        self.lambdas = np.stack([normalise(d) for d in np.atleast_2d(draws)])
        self.Y = np.stack([scalarise(lam, self.F, self.rho) for lam in self.lambdas], axis=1)
        self.mean = self.Y.mean(axis=0)  # mean::Data: the mean of each scalarised column
        return self.Y - self.mean

    def compute(self, X, F, draws) -> None:
        self.X = np.array(X, dtype=np.float64)
        self.F = np.array(F, dtype=np.float64)
        self.gp.set_data(self.X, self._columns(draws))
        self.gp.set_kernel(self.kernel_id, self.hparams, self.noise)
        self.gp.fit()

    def add_sample(self, x, f, draws) -> None:
        self.X = np.vstack([self.X, np.asarray(x, dtype=np.float64)[None, :]])
        self.F = np.vstack([self.F, np.asarray(f, dtype=np.float64)[None, :]])
        self.gp.append(self.X[-1], self._columns(draws))

    def query(self, Xq):
        """mu (M x q, the mean added) and sigma^2 (M)"""
        mu, s2 = self.gp.query(Xq)
        return mu + self.mean[None, :], s2

    def ucb(self, Xq, alpha: float):
        mu, s2 = self.query(Xq)
        return np.stack([O.ucb(mu[:, r], s2, alpha) for r in range(mu.shape[1])], axis=1)

    def ei(self, Xq, jitter: float = 0.0):
        """EI per column, f_max of column r = max over the samples of its mu (ei.hpp:100-108)"""
        f_max = self.query(self.X)[0].max(axis=0)
        mu, s2 = self.query(Xq)
        return np.stack([O.ei(mu[:, r], s2, f_max[r], jitter) for r in range(mu.shape[1])], axis=1)
