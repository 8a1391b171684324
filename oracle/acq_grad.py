"""Candidate gradients of mu, sigma^2, UCB / GP_UCB and EI in NumPy / SciPy: the formulas of limbo_b200/csrc/query_grad.cu over a
factor L and alpha (the oracle's, OracleGP.get), with W = K^-1 K* from cho_solve.

TEST INFRASTRUCTURE ONLY: the product package limbo_b200/ never imports this."""
from __future__ import annotations

import math

import numpy as np
from scipy.linalg import cho_solve, solve_triangular
from scipy.special import erfc

K_SE_ARD, K_MATERN52, K_MATERN32, K_EXP = 0, 1, 2, 3
DBL_EPSILON = np.finfo(np.float64).eps


def staging(kernel_id, hparams, D):
    """(J, sf2, l): staged coordinates u = x @ J (SE-ARD: [diag(1/ell) | A], squared_exp_ard.hpp:109-148; identity otherwise)."""
    hp = np.asarray(hparams, dtype=np.float64)
    if kernel_id == K_SE_ARD:
        klam = (hp.size - 1 - D) // D
        A = hp[D:D + D * klam].reshape(klam, D).T  # A(i, j) = p[(j + 1) D + i]
        return np.hstack([np.diag(np.exp(-hp[:D])), A]), math.exp(2.0 * hp[-1]), 1.0
    return np.eye(D), math.exp(2.0 * hp[1]), math.exp(hp[0])


def kernel_and_coef(kernel_id, z, sf2, l):
    """k(z) and c(z) with dk(u, u_n)/du = c (u - u_n), z = |u - u_n|^2."""
    if kernel_id == K_SE_ARD:
        k = sf2 * np.exp(-0.5 * z)
        return k, -k
    if kernel_id == K_EXP:
        k = sf2 * np.exp(-0.5 * z / (l * l))
        return k, -k / (l * l)
    d = np.sqrt(z)
    if kernel_id == K_MATERN52:
        a = math.sqrt(5.0) / l
        e = np.exp(-a * d)
        return sf2 * (1 + a * d + a * a * z / 3.0) * e, -sf2 * (a * a / 3.0) * (1 + a * d) * e
    a = math.sqrt(3.0) / l
    e = np.exp(-a * d)
    return sf2 * (1 + a * d) * e, -sf2 * a * a * e


def query_grad(kernel_id, hparams, noise, X, L, alpha, Xq):
    """mu (M x P, without mean), sigma^2 (M, clamped + noise), grad mu of the first output (M x D), grad sigma^2 (M x D, 0 where the
    clamp is active) and the per-candidate magnitude sum_n |g_n| (|alpha_n0| + 2 |W_nc|) (M x D) the device's error is bounded by."""
    X, Xq = np.atleast_2d(X), np.atleast_2d(Xq)
    alpha = np.asarray(alpha, dtype=np.float64).reshape(X.shape[0], -1)
    J, sf2, l = staging(kernel_id, hparams, X.shape[1])
    U, Uq = X @ J, Xq @ J
    diff = Uq[:, None, :] - U[None, :, :]                     # M x N x De
    z = np.einsum("mnd,mnd->mn", diff, diff)
    k, c = kernel_and_coef(kernel_id, z, sf2, l)               # M x N
    Ks = k.T                                                   # N x M
    mu = Ks.T @ alpha
    V = solve_triangular(L, Ks, lower=True)
    var = sf2 - np.einsum("nm,nm->m", V, V)
    clamped = var <= DBL_EPSILON
    s2 = np.where(clamped, 0.0, var) + noise
    W = cho_solve((L, True), Ks)                               # N x M
    g = c[:, :, None] * diff                                   # M x N x De
    dmu = np.einsum("mnd,n->md", g, alpha[:, 0]) @ J.T
    ds2 = -2.0 * np.einsum("mnd,nm->md", g, W) @ J.T
    ds2[clamped] = 0.0
    mag = np.einsum("mnd,mn->md", np.abs(g), np.abs(alpha[:, 0])[None, :] + 2.0 * np.abs(W.T)) @ np.abs(J.T)
    return mu, s2, dmu, ds2, mag


def ucb(mu0, s2, dmu, ds2, a):
    """UCB / GP_UCB value and gradient (ucb.hpp:89, gp_ucb.hpp:102): mu + a sqrt(s2)."""
    sq = np.sqrt(s2)
    with np.errstate(divide="ignore", invalid="ignore"):
        term = np.where((s2 > 0)[:, None], a * ds2 / (2.0 * sq)[:, None], 0.0)
    return mu0 + a * sq, dmu + term


def ei(mu0, s2, dmu, ds2, f_max, jitter=0.0):
    """EI value and gradient (ei.hpp:85-116), f_max and the jitter fixed; 0 where sigma < 1e-10."""
    sigma = np.sqrt(s2)
    live = ~(sigma < 1e-10)
    sg = np.where(live, sigma, 1.0)
    X = mu0 - f_max - jitter
    Z = X / sg
    phi = np.exp(-0.5 * Z * Z) / math.sqrt(2.0 * math.pi)
    Phi = 0.5 * erfc(-Z / math.sqrt(2.0))
    val = np.where(live, X * Phi + sg * phi, 0.0)
    grad = Phi[:, None] * dmu + phi[:, None] * ds2 / (2.0 * sg)[:, None]
    return val, np.where(live[:, None], grad, 0.0)
