"""NumPy restatement of the batched CMA-ES of limbo_b200/csrc/cmaes.cu (DESIGN.md §4.15): (mu/mu_w, lambda)-CMA-ES with the
active covariance update, in the default setting of Hansen, "The CMA Evolution Strategy: A Tutorial" (arXiv:1604.00772, Table 1
and Fig. 6), sampling through the Cholesky factor A of C.  It is not a port of libcmaes.  R independent instances advance in
lockstep; one generation of all of them is one call of the scoring callable on R * lambda candidates."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from limbo_b200 import synth

MAX_D, MAX_LAMBDA = 64, 256


@dataclass
class Constants:
    D: int
    lam: int
    mu: int
    w: np.ndarray        # lambda recombination weights: mu positive (sum 1), then the scaled negative ones
    mueff: float
    mueff_neg: float
    cs: float
    ds: float
    cc: float
    c1: float
    cmu: float
    chi: float           # E||N(0, I)||
    alpha_mu_neg: float
    alpha_mueff_neg: float
    alpha_posdef_neg: float


def default_lambda(D: int) -> int:
    return 4 + int(math.floor(3.0 * math.log(D)))


def constants(D: int, lam: int = 0) -> Constants:
    """The tutorial's default strategy parameters (Table 1) for dimension D and population lam (<= 0: 4 + floor(3 ln D))."""
    lam = lam if lam > 0 else default_lambda(D)
    mu = lam // 2
    i = np.arange(1, lam + 1, dtype=np.float64)
    wp = math.log((lam + 1) / 2.0) - np.log(i)
    pos, neg = wp[:mu], wp[mu:]
    mueff = pos.sum() ** 2 / (pos * pos).sum()
    sneg = np.abs(neg).sum()
    mueff_neg = neg.sum() ** 2 / (neg * neg).sum() if sneg > 0 else 0.0
    n = float(D)
    cc = (4.0 + mueff / n) / (n + 4.0 + 2.0 * mueff / n)
    cs = (mueff + 2.0) / (n + mueff + 5.0)
    c1 = 2.0 / ((n + 1.3) ** 2 + mueff)
    # c_mu as in arXiv:1604.00772v1 (2016), Table 1, alpha_cov = 2; later revisions add 1/4 to the numerator.  cmaes.cu states
    # the same form.
    cmu = min(1.0 - c1, 2.0 * (mueff - 2.0 + 1.0 / mueff) / ((n + 2.0) ** 2 + mueff))
    ds = 1.0 + 2.0 * max(0.0, math.sqrt((mueff - 1.0) / (n + 1.0)) - 1.0) + cs
    a_mu = 1.0 + c1 / cmu if cmu > 0 else math.inf
    a_mueff = 1.0 + 2.0 * mueff_neg / (mueff + 2.0)
    a_posdef = (1.0 - c1 - cmu) / (n * cmu) if cmu > 0 else math.inf
    w = np.empty(lam)
    w[:mu] = pos / pos.sum()
    w[mu:] = min(a_mu, a_mueff, a_posdef) / sneg * neg if sneg > 0 else 0.0
    chi = math.sqrt(n) * (1.0 - 1.0 / (4.0 * n) + 1.0 / (21.0 * n * n))
    return Constants(D, lam, mu, w, mueff, mueff_neg, cs, ds, cc, c1, cmu, chi, a_mu, a_mueff, a_posdef)


# ---- Hansen's linear-quadratic box transform on [lb, ub] ----------------------------------------------------------------------
def _widths(lb: float, ub: float):
    return min((ub - lb) / 2.0, (1.0 + abs(lb)) / 20.0), min((ub - lb) / 2.0, (1.0 + abs(ub)) / 20.0)


def transform(x, lb: float = 0.0, ub: float = 1.0) -> np.ndarray:
    """T: genotype -> phenotype, onto [lb, ub], the identity on [lb + al, ub - au]."""
    x = np.array(x, dtype=np.float64, copy=True)
    al, au = _widths(lb, ub)
    r = 2.0 * (ub - lb + al + au)
    xlow, xup = lb - 2.0 * al - (ub - lb) / 2.0, ub + 2.0 * au + (ub - lb) / 2.0
    lo = x < xlow
    x[lo] += r * (1.0 + np.floor((xlow - x[lo]) / r))
    hi = x > xup
    x[hi] -= r * (1.0 + np.floor((x[hi] - xup) / r))
    lo = x < lb - al
    x[lo] += 2.0 * (lb - al - x[lo])
    hi = x > ub + au
    x[hi] -= 2.0 * (x[hi] - ub - au)
    lo = x < lb + al
    x[lo] = lb + (x[lo] - lb + al) ** 2 / (4.0 * al)
    hi = x > ub - au
    x[hi] = ub - (x[hi] - ub - au) ** 2 / (4.0 * au)
    return x


def inverse(y, lb: float = 0.0, ub: float = 1.0) -> np.ndarray:
    """T^-1 on [lb, ub] (a point outside is clipped first): the genotype in [lb - al, ub + au] that T maps to y."""
    y = np.clip(np.array(y, dtype=np.float64, copy=True), lb, ub)
    al, au = _widths(lb, ub)
    lo = y < lb + al
    y[lo] = lb - al + 2.0 * np.sqrt(al * (y[lo] - lb))
    hi = y > ub - au
    y[hi] = ub + au - 2.0 * np.sqrt(au * (ub - y[hi]))
    return y


# ---- the draws ----------------------------------------------------------------------------------------------------------------
def normals(seed: int, g: int, R: int, lam: int, D: int) -> np.ndarray:
    """z (R x lam x D) of generation g: with c = ((g R + r) lam + k) D + d and u(i) = synth.uniform(seed, ., i),
    z = sqrt(-2 ln(1 - u(2c))) cos(2 pi u(2c + 1))."""
    n = R * lam * D
    u = synth.uniform(seed, 2 * n, 2 * g * n)
    return (np.sqrt(-2.0 * np.log(1.0 - u[0::2])) * np.cos(2.0 * np.pi * u[1::2])).reshape(R, lam, D)


# ---- one search -----------------------------------------------------------------------------------------------------------------
class Search:
    """R instances from the phenotypes `starts` (R x D).  step(score) runs one generation, score being a callable from an
    n x D array of phenotypes to n values (maximised)."""

    def __init__(self, starts, lam: int = 0, sigma0: float = 0.5, tolx: float = 1e-12, seed: int = 0, bounded: bool = True):
        starts = np.atleast_2d(np.asarray(starts, dtype=np.float64))
        self.R, self.D = starts.shape
        self.k = constants(self.D, lam)
        self.tolx, self.seed, self.bounded = float(tolx), int(seed), bool(bounded)
        self.g = 0
        self.m = inverse(starts) if bounded else starts.copy()
        self.sigma = np.full(self.R, float(sigma0))
        self.C = np.tile(np.eye(self.D), (self.R, 1, 1))
        self.A = self.C.copy()
        self.ps = np.zeros((self.R, self.D))
        self.pc = np.zeros((self.R, self.D))
        self.stopped = np.zeros(self.R, dtype=bool)
        self.best_val = np.full(self.R, -np.inf)
        self.best_x = np.clip(starts, 0.0, 1.0) if bounded else starts.copy()
        self.last_x = None
        self.last_vals = None

    def phenotype(self, x):
        return transform(x) if self.bounded else x

    def ask(self):
        """(z, y, phenotypes) of the current generation, each R x lam x D"""
        k = self.k
        z = normals(self.seed, self.g, self.R, k.lam, self.D)
        y = np.einsum("rij,rkj->rki", self.A, z)
        x = self.m[:, None, :] + self.sigma[:, None, None] * y
        return z, y, self.phenotype(x)

    def step(self, score) -> None:
        k, D = self.k, self.D
        z, y, X = self.ask()
        vals = np.asarray(score(X.reshape(-1, D)), dtype=np.float64).reshape(self.R, k.lam)
        self.last_x, self.last_vals = X, vals
        for r in range(self.R):
            if not self.stopped[r]:
                self._tell(r, z[r], y[r], X[r], vals[r])
        self.g += 1

    @staticmethod
    def ranking(vals) -> np.ndarray:
        """offspring indices by value, descending; NaN last; ties to the lower index"""
        key = np.where(np.isnan(vals), -np.inf, vals)
        nan = np.isnan(vals)
        return np.lexsort((np.arange(len(vals)), -key, nan))

    def _tell(self, r, z, y, X, vals) -> None:
        k, D = self.k, self.D
        order = self.ranking(vals)
        j = order[0]
        if vals[j] > self.best_val[r]:
            self.best_val[r], self.best_x[r] = vals[j], X[j].copy()
        zs, ys = z[order], y[order]
        w = k.w
        yw = w[:k.mu] @ ys[:k.mu]
        zw = w[:k.mu] @ zs[:k.mu]
        self.m[r] = self.m[r] + self.sigma[r] * yw
        self.ps[r] = (1.0 - k.cs) * self.ps[r] + math.sqrt(k.cs * (2.0 - k.cs) * k.mueff) * zw
        nps = float(np.sqrt(self.ps[r] @ self.ps[r]))
        hs = 1.0 if nps / math.sqrt(1.0 - (1.0 - k.cs) ** (2 * (self.g + 1))) < (1.4 + 2.0 / (D + 1.0)) * k.chi else 0.0
        self.pc[r] = (1.0 - k.cc) * self.pc[r] + hs * math.sqrt(k.cc * (2.0 - k.cc) * k.mueff) * yw
        wo = w.copy()
        nz2 = (zs * zs).sum(axis=1)
        wo[k.mu:] = w[k.mu:] * D / nz2[k.mu:]
        coef = 1.0 + k.c1 * (1.0 - hs) * k.cc * (2.0 - k.cc) - k.c1 - k.cmu * w.sum()
        C = coef * self.C[r] + k.c1 * np.outer(self.pc[r], self.pc[r]) + k.cmu * (ys.T * wo) @ ys
        C = 0.5 * (C + C.T)
        self.sigma[r] *= math.exp(k.cs / k.ds * (nps / k.chi - 1.0))
        self.C[r] = C
        try:
            self.A[r] = np.linalg.cholesky(C)
        except np.linalg.LinAlgError:
            self.stopped[r] = True
            return
        if not (np.isfinite(self.sigma[r]) and self.sigma[r] * math.sqrt(np.max(np.diag(C))) >= self.tolx):
            self.stopped[r] = True

    def best(self):
        """(best phenotype, its value) over every instance and generation; ties to the lower instance"""
        i = int(np.argmax(np.where(np.isnan(self.best_val), -np.inf, self.best_val)))
        return self.best_x[i].copy(), float(self.best_val[i])


def run(score, starts, generations: int, **kw) -> tuple[np.ndarray, float, int]:
    """A whole search as lb_acq_cmaes runs it: every instance stops after `generations` generations, or earlier (tolx, a failed
    factorisation); the live instances are counted after every 8th generation.  Returns (best_x, best_val, evaluations)."""
    s = Search(starts, **kw)
    for g in range(generations):
        s.step(score)
        if (g + 1) % 8 == 0 and s.stopped.all():
            break
    bx, bv = s.best()
    return bx, bv, s.g * s.R * s.k.lam
