"""NumPy fp64 restatement of the reference's experimental::model::SPGP (src/limbo/experimental/model/spgp.hpp), written from
its equations in the reference's order.  Kept quirks (DESIGN.md §8):
  * w = [xb (M*D, read column-major), log b (D), log c, log sig]; b is the inverse squared length scale (:94-101);
  * the initial pseudo-inputs are written row-major into the column-major xb block (:420-421);
  * the value's (n - _m) / 2 * log(sig) is an integer division (:491);
  * ep comes from the unscaled V, sumVsq from the scaled one, and the D-loop uses the scaled K (:480-483, :513).
Test infrastructure only: the product computes all of this on the device (limbo_b200/csrc/spgp.cu)."""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg as sla


def n_params(M: int, D: int) -> int:
    return (M + 1) * D + 2


def unpack(w, M: int, D: int):
    """HyperParams(w, m, dim_in) (:94-101): xb (M x D), b (D), c, sig."""
    w = np.asarray(w, dtype=np.float64)
    assert w.size == n_params(M, D)
    xb = w[:M * D].reshape(D, M).T.copy()  # Eigen's resize keeps the column-major storage
    b = np.exp(w[M * D:(M + 1) * D])
    return xb, b, math.exp(w[(M + 1) * D]), math.exp(w[(M + 1) * D + 1])


def n_pseudo(N: int, samples_percent: float = 10.0, min_m: int = 1) -> int:
    """_update_m (:381-387): floor(samples_percent * N / 100), at least min_m."""
    m = int(samples_percent * N / 100)
    return max(m, min_m)


def init_w(X, y_zm, M: int, perm) -> np.ndarray:
    """_optimize_hyperparams' initial vector (:414-426) for a given permutation of the sample indices."""
    X = np.asarray(X, dtype=np.float64)
    N, D = X.shape
    w = np.empty(n_params(M, D))
    for i in range(M):  # row-major into the column-major xb block, as the reference does
        w[i * D:(i + 1) * D] = X[perm[i]]
    w[M * D:(M + 1) * D] = -2.0 * np.log((X.max(axis=0) - X.min(axis=0)) / 2.0)
    y = np.asarray(y_zm, dtype=np.float64).reshape(-1)
    w[(M + 1) * D] = math.log(np.mean(y ** 2))
    w[(M + 1) * D + 1] = math.log(np.mean(y ** 2 / 4.0))
    return w


def _lower_solve(L, B):
    return sla.solve_triangular(L, B, lower=True)


def _upper_solve(U, B):
    return sla.solve_triangular(U, B, lower=False)


def likelihood(w, X, y_zm, M: int, jitter: float, grad: bool = True, fix_integer_division: bool = False):
    """_likelihood(w, grad) with inverse = true (:446-451, :453-580): (-fw, -dfw).  fix_integer_division uses (n - m) / 2 in
    floating point instead (the value the reference means; tests pin the difference)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y_zm, dtype=np.float64).reshape(-1, 1)
    n, D = X.shape
    xb, b, c, sig = unpack(w, M, D)
    dl = jitter
    bs = np.sqrt(b)[None, :]
    xb = xb * bs
    x = X * bs
    Q = xb @ xb.T
    dq = np.diag(Q)
    Q = dq[:, None] + dq[None, :] - 2 * Q
    Q = np.exp(Q * -0.5) * c
    Q = Q + dl * np.eye(M)
    K = -2 * xb @ x.T + np.sum(x * x, axis=1)[None, :] + np.sum(xb * xb, axis=1)[:, None]
    K = np.exp(K * -0.5) * c
    L = np.linalg.cholesky(Q)
    V = _lower_solve(L, K)
    ep = 1 + (c - np.sum(V ** 2, axis=0)[:, None]) / sig
    se = np.sqrt(ep)
    K = K / se.T
    V = V / se.T
    y = y / se
    Lm = np.linalg.cholesky(sig * np.eye(M) + V @ V.T)
    invLmV = _lower_solve(Lm, V)
    bet = invLmV @ y
    half = (n - M) // 2 if not fix_integer_division else (n - M) / 2
    fw = (np.sum(np.log(np.diag(Lm))) + half * math.log(sig) + (y.T @ y - bet.T @ bet).item() / (2 * sig)
          + np.sum(np.log(ep)) / 2 + 0.5 * n * math.log(2 * math.pi))
    if not grad:
        return -fw, None
    Lt = L @ Lm
    B1 = _upper_solve(Lt.T, invLmV)
    b1 = _upper_solve(Lt.T, bet)
    invLV = _upper_solve(L.T, V)
    invL = np.linalg.inv(L)
    invQ = invL.T @ invL
    invLt = np.linalg.inv(Lt)
    invA = invLt.T @ invLt
    mu = (_upper_solve(Lm.T, bet).T @ V).T
    sumVsq = np.sum(V ** 2, axis=0)[:, None]
    bigsum = y * (bet.T @ invLmV).T / sig - np.sum(invLmV ** 2, axis=0)[:, None] / 2 - (y ** 2 + mu ** 2) / (2 * sig) + 0.5
    TT = invLV @ (invLV.T * bigsum)
    dfxb = np.empty((M, D))
    dfb = np.empty(D)
    for i in range(D):
        dnnQ = (xb[:, i:i + 1] - xb[:, i:i + 1].T) * Q
        dNnK = (-xb[:, i:i + 1] - (-x[:, i:i + 1]).T) * K
        epdot = dNnK * invLV * (-2 / sig)
        epPmod = -np.sum(epdot, axis=0)[:, None]
        col = (-(b1 * ((dNnK @ (y - mu)) / sig + dnnQ @ b1)) + np.sum((invQ - invA * sig) * dnnQ, axis=1)[:, None]
               + epdot @ bigsum - np.sum(dnnQ * TT, axis=1)[:, None] * (2 / sig))
        dfbi = ((((y - mu).T * (b1.T @ dNnK)) / sig + (epPmod * bigsum).T) @ x[:, i]).item()
        dNnK = dNnK * B1
        col = col + np.sum(dNnK, axis=1)[:, None]
        dfbi -= float(np.sum(dNnK, axis=0) @ x[:, i])
        col = col * math.sqrt(b[i])
        dfbi /= math.sqrt(b[i])
        dfbi += float(col[:, 0] @ xb[:, i]) / b[i]
        dfbi *= math.sqrt(b[i]) / 2
        dfxb[:, i] = col[:, 0]
        dfb[i] = dfbi
    epc = (c / ep - sumVsq - dl * np.sum(invLV ** 2, axis=0)[:, None]) / sig
    dfc = ((M + dl * np.trace(invQ - sig * invA) - sig * np.sum(invA * Q.T)) / 2 - (mu.T @ (y - mu)).item() / sig
           + (b1.T @ (Q - dl * np.eye(M)) @ b1).item() / 2 + (epc.T @ bigsum).item())
    dfsig = float(np.sum(bigsum / ep))
    dfw = np.concatenate([dfxb.T.reshape(-1), dfb, [dfc, dfsig]])  # dfxb flattened column-major (:568)
    return -fw, -dfw


def _kernel_matrix(p1, p2, b, c):
    """_compute_kernel_matrix (:612-628)."""
    bs = np.sqrt(b)[None, :]
    x1 = p1 * bs
    x2 = p2 * bs
    K = (-2 * x1 @ x2.T) + np.sum(x2 ** 2, axis=1)[None, :] + np.sum(x1 ** 2, axis=1)[:, None]
    return c * np.exp(K * -0.5)


class State:
    """What _compute(false) (:389-407) leaves behind at HyperParams(w)."""

    def __init__(self, w, X, y_zm, M: int, jitter: float):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y_zm, dtype=np.float64).reshape(-1, 1)
        N, D = X.shape
        self.xb, self.b, self.c, self.sig = unpack(w, M, D)
        km = _kernel_matrix(self.xb, self.xb, self.b, self.c) + np.eye(M) * jitter
        self.L = np.linalg.cholesky(km)
        kmn = _kernel_matrix(self.xb, X, self.b, self.c)
        V = _lower_solve(self.L, kmn)
        ep = np.ones((N, 1)) + (self.c - np.sum(V ** 2, axis=0)[:, None]) / self.sig
        es = np.sqrt(ep)
        V = V / es.T
        y = y / es
        self.Lm = np.linalg.cholesky(self.sig * np.eye(M) + V @ V.T)
        self.bet = _lower_solve(self.Lm, V @ y)[:, 0]

    def predict(self, Xq, optimized: bool = True):
        """_predict (:582-610) without mean(v): (mu - mean, sigma^2)."""
        K = _kernel_matrix(self.xb, np.asarray(Xq, dtype=np.float64), self.b, self.c)
        lst = _lower_solve(self.L, K)
        lmst = _lower_solve(self.Lm, lst)
        mu = self.bet @ lmst
        s2 = self.c - np.sum(lst ** 2, axis=0) + self.sig * np.sum(lmst ** 2, axis=0) + (self.sig if optimized else 0.0)
        return mu, s2


def ucb(mu, s2, alpha: float):
    return mu + alpha * np.sqrt(s2)
