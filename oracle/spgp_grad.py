"""NumPy fp64 candidate gradients of the reference's SPGP prediction (oracle/spgp.py's State, _predict of
src/limbo/experimental/model/spgp.hpp:582-610), which the reference does not provide.  With b the inverse squared length scales,
x~ = x o sqrt(b), x~b_m = xb_m o sqrt(b), k_m = c exp(-|x~ - x~b_m|^2 / 2), lst = L^-1 k, lmst = Lm^-1 lst and k(x, x) = c:
    grad mu      = -sqrt(b) o sum_m b1_m k_m (x~ - x~b_m),   b1 = L^-T Lm^-T bet
    grad sigma^2 =  2 sqrt(b) o sum_m u_m k_m (x~ - x~b_m),  u = L^-T (lst - sig Lm^-T lmst)
and the per-entry magnitude sqrt(b_d) sum_m k_m |x~_d - x~b_md| (|b1_m| + 2 |u_m|) that scales the rounding error of both sums.
Test infrastructure only: the product computes this on the device (limbo_b200/csrc/spgp.cu, lb_spgp_query_grad)."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

from .spgp import _kernel_matrix


def query_grad(st, Xq, optimized: bool = True):
    """(mu - mean, sigma^2, grad mu, grad sigma^2, magnitude) at the candidates Xq (Mq x D) of a oracle.spgp.State; the gradients
    and the magnitude are Mq x D."""
    Xq = np.atleast_2d(np.asarray(Xq, dtype=np.float64))
    sb = np.sqrt(st.b)
    K = _kernel_matrix(st.xb, Xq, st.b, st.c)  # M x Mq
    lst = sla.solve_triangular(st.L, K, lower=True)
    lmst = sla.solve_triangular(st.Lm, lst, lower=True)
    mu = st.bet @ lmst
    s2 = st.c - np.sum(lst ** 2, axis=0) + st.sig * np.sum(lmst ** 2, axis=0) + (st.sig if optimized else 0.0)
    b1 = sla.solve_triangular(st.L.T, sla.solve_triangular(st.Lm.T, st.bet, lower=False), lower=False)
    u = sla.solve_triangular(st.L.T, lst - st.sig * sla.solve_triangular(st.Lm.T, lmst, lower=False), lower=False)
    diff = (Xq * sb)[None, :, :] - (st.xb * sb)[:, None, :]  # M x Mq x D
    dmu = -sb * np.einsum("m,mq,mqd->qd", b1, K, diff)
    ds2 = 2.0 * sb * np.einsum("mq,mq,mqd->qd", u, K, diff)
    mag = sb * np.einsum("mq,mqd->qd", K * (np.abs(b1)[:, None] + 2.0 * np.abs(u)), np.abs(diff))
    return mu, s2, dmu, ds2, mag
