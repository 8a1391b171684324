"""Matrices with an exactly known Cholesky factor, numpy restatements of the kernel derivatives, and first-order
rounding-error bounds for the fp64 factorisation, inverse, solves and query (tests/test_linalg_exact_host.py,
tests/test_gpu_linalg_exact.py).

K = L0 L0^T with L0 integer lower-triangular: a diagonal in [2^11, 2^12], strictly-lower entries in [-8, 8].  Every
entry of K is an integer below 2^53, so any fp64 BLAS forms it exactly and its Cholesky factor is exactly L0.  The
right-hand side is Y = K A0 with A0 = integers * 2^-14 (a power-of-two scale keeps Y exact), so the solve's truth is
exactly A0, and log det K = 2 sum log L0_ii.  K is well conditioned (kappa_2 is a small number, asserted per case), so
every tile of L, L^-1 and alpha carries weight and the bars below come from rounding-error analysis alone:

  gamma_n = n u / (1 - n u), u = 2^-53 (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Lemma 3.1).
  Cholesky (Thm 10.3):  L^ L^T = K + dK, |dK| <= gamma_{n+1} |L^||L^T|.  The device forms the off-diagonal blocks by
      multiplying with the explicit inverse of the 128 x 128 diagonal block, which multiplies the backward error by
      at most kappa_inf of that block (Du Croz and Higham, 1992): c_blk = max_k kappa_inf(L0_kk).
  Forward error of L (Sun, 1991 / Higham Thm 10.8):  ||dL||_F <= kappa_2(K) ||L||_2 ||dK||_F / ||K||_2.
  Solve (Thm 10.4):  (K + dK) x^ = b, |dK| <= gamma_{3n+1} |L^||L^T|  ->  ||dx|| <= kappa_2(K) ||dK||_2 / ||K||_2 ||x||.
  Inverse (Higham section 14.2): ||dX||_F <= kappa_2(K) (backward error) ||K^-1||_F, for the device and the LAPACK
      reference alike (both terms are added).
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -53
TILE = 128
A0_SCALE = 2.0 ** -14
KERNELS = (0, 1, 2, 3)  # SE-ARD, Matern 5/2, Matern 3/2, Exp (limbo_b200._lib.KERNEL_*)
KERNEL_NAMES = {0: "se_ard", 1: "matern52", 2: "matern32", 3: "exp"}


def gamma(n: float) -> float:
    nu = n * U
    assert nu < 1.0
    return nu / (1.0 - nu)


# ---------------------------------------------------------------------------------------------------------------------
# exact cases
# ---------------------------------------------------------------------------------------------------------------------
class ExactCase:
    """K = L0 L0^T (exact), Y = K A0 (exact), host reference quantities for the bounds."""

    def __init__(self, N: int, P: int, seed: int):
        rng = np.random.default_rng(seed)
        self.N, self.P, self.seed = N, P, seed
        L0 = np.tril(rng.integers(-8, 9, size=(N, N)).astype(np.float64), -1)
        L0[np.diag_indices(N)] = rng.integers(2 ** 11, 2 ** 12 + 1, size=N).astype(np.float64)
        self.L0 = L0
        self.K = L0 @ L0.T
        self.A0 = np.asfortranarray(rng.integers(-8, 9, size=(N, P)).astype(np.float64) * A0_SCALE)
        self.Y = np.asfortranarray(self.K @ self.A0)
        self.logdet = 2.0 * math.fsum(math.log(v) for v in np.diag(L0))
        self._ref = None

    @property
    def T(self) -> int:
        return max(1, -(-self.N // TILE))

    def ref(self):
        """Host reference quantities (computed once): kappa_2(K), ||K||_2, ||K^-1||_2, ||L0||_F, || |L0||L0^T| ||_F,
        c_blk, and K^-1 from LAPACK dpotri on the exact factor."""
        if self._ref is None:
            import scipy.linalg as sl
            ev = sl.eigh(self.K, eigvals_only=True, driver="evr", subset_by_index=[0, 0]), \
                sl.eigh(self.K, eigvals_only=True, driver="evr", subset_by_index=[self.N - 1, self.N - 1])
            lmin, lmax = float(ev[0][0]), float(ev[1][0])
            absL = np.abs(self.L0)
            kinv, info = sl.lapack.dpotri(self.L0, lower=1)
            assert info == 0
            kinv = np.tril(kinv)
            kinv = kinv + np.tril(kinv, -1).T
            self._ref = dict(kappa=lmax / lmin, norm_k=lmax, norm_kinv=1.0 / lmin, abs_llt_f=float(np.linalg.norm(absL @ absL.T)),
                             c_blk=block_kappa(self.L0), kinv=kinv)
        return self._ref

    def with_bad_pivot(self, p: int) -> np.ndarray:
        """K with K_pp lowered so that the Schur complement at p is exactly -K_pp / 2: dpotrf stops there (info p + 1).
        K_pp - sum_k<p L0_pk^2 = L0_pp^2, so K'_pp = K_pp - L0_pp^2 - K_pp / 2 (a half-integer: exact)."""
        Kb = self.K.copy()
        Kb[p, p] = self.K[p, p] - self.L0[p, p] ** 2 - 0.5 * self.K[p, p]
        return Kb


def block_kappa(L: np.ndarray) -> float:
    """max over the 128 x 128 diagonal blocks of kappa_inf(L_kk) (the triangular blocks the device inverts explicitly)."""
    import scipy.linalg as sl
    N = L.shape[0]
    c = 1.0
    for k0 in range(0, N, TILE):
        B = L[k0:k0 + TILE, k0:k0 + TILE]
        Bi = sl.solve_triangular(B, np.eye(B.shape[0]), lower=True)
        c = max(c, np.abs(B).sum(1).max() * np.abs(Bi).sum(1).max())
    return float(c)


def bound_L(case: ExactCase) -> float:
    """Frobenius bound on L^ - L0."""
    r = case.ref()
    n = case.N
    dK = case_cblk(case) * gamma(n + 1) * r["abs_llt_f"]
    return r["kappa"] * math.sqrt(r["norm_k"]) * dK / r["norm_k"]


def case_cblk(case: ExactCase) -> float:
    return case.ref()["c_blk"]


def bound_alpha(case: ExactCase) -> np.ndarray:
    """2-norm bound on alpha^ - A0, per column."""
    r = case.ref()
    n = case.N
    rel = r["kappa"] * case_cblk(case) * gamma(3 * n + 1) * r["abs_llt_f"] / r["norm_k"]
    return rel * np.linalg.norm(case.A0, axis=0)


def bound_logdet(case: ExactCase) -> float:
    """|logdet^ - logdet| from lb_log_lik with alpha = 0: the diagonal of L (through the L bound), the logs and the sum,
    and the rounding of 0.5 N log(2 pi) and of -2 * loglik on the host."""
    n = case.N
    dmin = float(np.diag(case.L0).min())
    s = float(np.abs(2.0 * np.log(np.diag(case.L0))).sum())
    return 2.0 * math.sqrt(n) * bound_L(case) / dmin + gamma(n + 4) * (s + n * math.log(2 * math.pi))


def bound_kinv(case: ExactCase) -> float:
    """Frobenius bound on K^-1^ - K^-1 (device + LAPACK reference)."""
    r = case.ref()
    n = case.N
    back = case_cblk(case) * gamma(3 * n + 1) * r["abs_llt_f"] / r["norm_k"]
    return 2.0 * r["kappa"] * back * math.sqrt(n) * r["norm_kinv"]


def worst_tile(err: np.ndarray) -> str:
    """The 128 x 128 tile holding the largest |err| (for failure messages)."""
    e = np.abs(np.atleast_2d(err))
    if e.size == 0:
        return "empty"
    i, j = np.unravel_index(int(np.nanargmax(np.where(np.isnan(e), np.inf, e))), e.shape)
    return f"max |err| {e[i, j]:.3e} at ({i}, {j}) = tile ({i // TILE}, {j // TILE})"


# shapes of the exact-factor cases: T = 1 .. 13 (every quad and trtri tail), 15 .. 17, 24, 31 .. 33 (the panel query's
# ragged 16-tile super-blocks); N mod 128 cycles through {0, 1, 127} (all three at T = 5, 9, 17, 33); N = 1 at T = 1
T_LIST = list(range(1, 14)) + [15, 16, 17, 24, 31, 32, 33]
THREE_EDGES = (5, 9, 17, 33)
QUERY_T = (1, 2, 15, 16, 17, 31, 32, 33)


def exact_shapes():
    """(N, P, seed) of every exact-factor case, P cycling through 1, 3, 5."""
    out = []
    for i, T in enumerate(T_LIST):
        edges = (128 * T, 128 * (T - 1) + 1, 128 * T - 1)
        Ns = list(edges) if T in THREE_EDGES else [edges[T % 3]]
        for j, N in enumerate(Ns):
            out.append((N, (1, 3, 5)[(i + j) % 3], 1000 + 10 * i + j))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# kernels: values and derivatives (the formulas of oracle/limbo_oracle.hpp, vectorised)
# ---------------------------------------------------------------------------------------------------------------------
def kernel_params(kid: int, D: int, rng) -> np.ndarray:
    if kid == 0:
        return np.concatenate([rng.uniform(-0.7, 0.3, D), [rng.uniform(-0.3, 0.3)]])
    return np.array([rng.uniform(-1.0, 0.0), rng.uniform(-0.3, 0.3)])


def _sqdist(X1, X2, scale=None):
    """Squared distances from the coordinate differences (no Gram-matrix trick, which cancels for close points)."""
    A = X1 if scale is None else X1 * scale
    B = X2 if scale is None else X2 * scale
    z = np.zeros((X1.shape[0], X2.shape[0]))
    for d in range(A.shape[1]):
        q = A[:, d, None] - B[None, :, d]
        z += q * q
    return z


def kernel_matrix(kid: int, p: np.ndarray, X1: np.ndarray, X2: np.ndarray) -> np.ndarray:
    """k(x1, x2) without noise, as in Kernel::kernel of each functor."""
    if kid == 0:
        D = X1.shape[1]
        sf2 = math.exp(2 * p[D])
        return sf2 * np.exp(-0.5 * _sqdist(X1, X2, np.exp(-p[:D])))
    l, sf2 = math.exp(p[0]), math.exp(2 * p[1])
    s = _sqdist(X1, X2)
    if kid == 3:
        return sf2 * np.exp(-0.5 * s / (l * l))
    r = np.sqrt(s)
    if kid == 1:
        t1 = math.sqrt(5.0) * r / l
        t2 = 5.0 * s / (3.0 * l * l)
        return sf2 * (1.0 + t1 + t2) * np.exp(-t1)
    t = math.sqrt(3.0) * r / l
    return sf2 * (1.0 + t) * np.exp(-t)


def kernel_grads(kid: int, p: np.ndarray, X1: np.ndarray, X2: np.ndarray):
    """Yields dk(x1, x2) / d theta_q for every hyper-parameter q (log ell_d / log l, then log sigma_f), as matrices."""
    if kid == 0:
        D = X1.shape[1]
        sf2 = math.exp(2 * p[D])
        inv = np.exp(-p[:D])
        k = sf2 * np.exp(-0.5 * _sqdist(X1, X2, inv))
        for d in range(D):
            q = (X1[:, d, None] - X2[None, :, d]) * inv[d]
            yield q * q * k
        yield 2.0 * k
        return
    l, sf2 = math.exp(p[0]), math.exp(2 * p[1])
    s = _sqdist(X1, X2)
    if kid == 3:
        r = s / (l * l)
        k = sf2 * np.exp(-0.5 * r)
        yield r * k
        yield 2.0 * k
        return
    d = np.sqrt(s)
    if kid == 1:
        t1 = math.sqrt(5.0) * d / l
        t2 = 5.0 * s / (3.0 * l * l)
        e = np.exp(-t1)
        yield sf2 * (e * t1 * (1.0 + t1 + t2) + (-t1 - 2.0 * t2) * e)
        yield 2.0 * sf2 * (1.0 + t1 + t2) * e
        return
    t = math.sqrt(3.0) * d / l
    e = np.exp(-t)
    yield sf2 * (-t * e + (1.0 + t) * t * e)
    yield 2.0 * sf2 * (1.0 + t) * e


def kernel_eval_err(kid: int, p: np.ndarray, xmax: float, D: int) -> float:
    """Absolute bound on the fp64 evaluation error of one kernel value or derivative, inputs in [-xmax, xmax]^D.
    Every formula is sf^2 * (polynomial of degree <= 3 in rho) * exp(-rho) of the squared distance z, Lipschitz in z
    with constant <= sf^2 (1 + a^2)(1 + rho)^2 (a: the scale of z inside rho); z itself is a sum of D squared differences
    of (pre-scaled) coordinates, so |dz| <= gamma_{D+3} zb with zb the largest sum of (|x_d| + |y_d|)^2 / scale_d^2."""
    if kid == 0:
        sf2 = math.exp(2 * p[D])
        zb = float(((2.0 * xmax * np.exp(-p[:D])) ** 2).sum())
        a2, rho = 1.0, 0.5 * zb
    else:
        l, sf2 = math.exp(p[0]), math.exp(2 * p[1])
        zb = D * (2.0 * xmax) ** 2
        if kid == 3:
            a2 = 1.0 / (l * l)
            rho = 0.5 * a2 * zb
        else:
            a2 = (5.0 if kid == 1 else 3.0) / (l * l)
            rho = math.sqrt(a2 * zb)
    return sf2 * ((1.0 + a2) * (1.0 + rho) ** 2 * gamma(D + 3) * zb + gamma(32) * (1.0 + rho) ** 3 * (1.0 + zb))


def grad_reference(kid, p, X, alpha, kinv, noise, optimize_noise):
    """0.5 sum_ij (alpha alpha^T - K^-1)_ij dk_ij / d theta_q (gp.hpp:285-311), and the matching sums of |W| |dk| and
    ||dk||_F per hyper-parameter for the bound."""
    W = alpha @ alpha.T - kinv
    g, absum, fro = [], [], []
    for dk in kernel_grads(kid, p, X, X):
        g.append(0.5 * float((W * dk).sum()))
        absum.append(0.5 * float((np.abs(W) * np.abs(dk)).sum()))
        fro.append(float(np.linalg.norm(dk)))
    if optimize_noise:
        dn = 2.0 * noise
        g.append(0.5 * float(np.trace(W)) * dn)
        absum.append(0.5 * float(np.abs(np.diag(W)).sum()) * dn)
        fro.append(dn * math.sqrt(X.shape[0]))
    return np.array(g), np.array(absum), np.array(fro)


def bound_grad(case: ExactCase, kid, p, X, absum, fro, da_bound, dkinv_bound) -> np.ndarray:
    """|g^ - g| per hyper-parameter: ||dW||_F ||dk_q||_F (dW from the alpha and K^-1 bounds: alpha alpha^T moves by at
    most 2 ||d alpha|| ||alpha|| per output), the products and the sum of N^2 terms on the device and on the host, and
    the evaluation error of dk (kernel_eval_err) times sum |W|."""
    n = case.N
    na = np.linalg.norm(case.A0, axis=0)
    dW = float(2.0 * (da_bound * na).sum() + dkinv_bound)
    W = case.A0 @ case.A0.T - case.ref()["kinv"]
    wsum = float(np.abs(W).sum())
    ev = kernel_eval_err(kid, p, float(np.abs(X).max()), X.shape[1])
    return 0.5 * dW * fro + 2.0 * gamma(n * n + case.P + 8) * absum + 0.5 * ev * wsum


# ---------------------------------------------------------------------------------------------------------------------
# query on a loaded factor
# ---------------------------------------------------------------------------------------------------------------------
class QueryCase:
    """A random lower-triangular L = c (I + E) with ||E||_1, ||E||_inf <= 1/4 (so ||E||_2 <= 1/4 and kappa_2(L) <= 5/3),
    training points X in [0,1]^D and alpha random; c is chosen per candidate set so that max ||L^-1 k*||^2 = sf^2 / 2."""

    def __init__(self, N: int, D: int, P: int, seed: int):
        rng = np.random.default_rng(seed)
        self.N, self.D, self.P = N, D, P
        self.E = np.tril(rng.uniform(-1.0, 1.0, size=(N, N)), -1) * (0.25 / N)
        self.X = rng.uniform(0.0, 1.0, size=(N, D))
        self.alpha = np.asfortranarray(rng.uniform(-1.0, 1.0, size=(N, P)))
        self.rng = rng

    def norm_E(self) -> float:
        return math.sqrt(np.abs(self.E).sum(0).max() * np.abs(self.E).sum(1).max())

    def reference(self, kid, p, noise, Xq):
        """(L, mu, sigma2, V, K*) for candidates Xq with c fitted to this candidate set."""
        import scipy.linalg as sl
        Ks = kernel_matrix(kid, p, self.X, Xq)
        A = np.eye(self.N) + self.E
        V1 = sl.solve_triangular(A, Ks, lower=True)
        sf2 = math.exp(2 * p[-1])
        c = math.sqrt(2.0 * float((V1 * V1).sum(0).max()) / sf2)
        L = np.asfortranarray(c * A)
        V = V1 / c
        mu = Ks.T @ self.alpha
        s2 = sf2 - (V * V).sum(0) + noise
        return L, mu, s2, V, Ks

    def grad_reference(self, kid, p, noise, Xq, L=None) -> dict:
        """mu, sigma^2 (s2), grad mu of output 0 (dmu), grad sigma^2 (ds2), V = L^-1 K* and W = L^-T V of candidates Xq, with
        two triangular solves in staged coordinates u = x J (oracle/acq_grad.staging: SE-ARD's Lambda columns enter only
        through J); also the factor L, K* (Ks) and the pairs' differences Q, distances d and coefficients c for grad_bounds.
        L: c (I + E) with c fitted to this candidate set as in reference(), unless given."""
        import scipy.linalg as sl
        J, _, _, Q, d, k, cc = _staged_pairs(kid, p, self.X, Xq)
        sf2 = staging(kid, p, self.D)[1]
        if L is None:
            V1 = sl.solve_triangular(np.eye(self.N) + self.E, k, lower=True)
            c = math.sqrt(2.0 * float((V1 * V1).sum(0).max()) / sf2)
            L = np.asfortranarray(c * (np.eye(self.N) + self.E))
        V = sl.solve_triangular(L, k, lower=True)
        W = sl.solve_triangular(L, V, lower=True, trans="T")
        a0 = self.alpha[:, 0]
        return dict(L=L, Ks=k, V=V, W=W, Q=Q, d=d, c=cc,
                    mu=k.T @ self.alpha, s2=sf2 - (V * V).sum(0) + noise,
                    dmu=np.stack([(cc * q).T @ a0 for q in Q], axis=1) @ J.T,
                    ds2=np.stack([-2.0 * ((cc * q) * W).sum(0) for q in Q], axis=1) @ J.T)


def bound_mu(kid, p, Ks, alpha, xmax, D):
    """|mu^ - mu| per candidate and output: the dot product (device and host) and the kernel evaluation."""
    n = Ks.shape[0]
    ev = kernel_eval_err(kid, p, xmax, D)
    return 2.0 * gamma(n + 2) * (np.abs(Ks).T @ np.abs(alpha)) + ev * np.abs(alpha).sum(0)[None, :]


def bound_s2(kid, p, V, c, normE, xmax, D, noise):
    """|sigma2^ - sigma2| per candidate: the triangular solve (backward error gamma_n |L| times c_blk <= kappa_inf of a
    block of I + E, <= (5/4)/(3/4)), its forward error through kappa_2(L) <= (1+|E|)/(1-|E|), the sum of squares, the
    kernel evaluation through ||L^-1|| <= 1/(c (1 - |E|)), and the final subtraction and addition."""
    n = V.shape[0]
    sf2 = math.exp(2 * p[-1])
    kap = (1.0 + normE) / (1.0 - normE)  # kappa_2(L), and an upper bound of || |L| ||_2 / ||L||_2 * kappa_inf(L_kk)
    v2 = (V * V).sum(0)
    nv = np.sqrt(v2)
    ev = kernel_eval_err(kid, p, xmax, D)
    dv = kap * kap * gamma(n) * nv + ev * math.sqrt(n) / (c * (1.0 - normE))
    # device and host reference each: 2 ||v|| ||dv|| + the sum of squares; then sf2 - s + noise
    return 2.0 * (2.0 * nv * dv + gamma(n + 2) * v2) + 4.0 * U * (sf2 + v2 + abs(noise))


# ---------------------------------------------------------------------------------------------------------------------
# candidate gradients on a loaded factor (lb_query_grad / lb_acq_grad)
# ---------------------------------------------------------------------------------------------------------------------
def staging(kid, p, D):
    """(J, sf2, l, a): staged coordinates u = x J as oracle/acq_grad.staging (SE-ARD: [diag(1/ell) | Lambda], the identity
    otherwise), and the scale a of the distance d = |u - u_n| in the exponent (Matern: sqrt(5)/l, sqrt(3)/l)."""
    from oracle import acq_grad as AG
    J, sf2, l = AG.staging(kid, p, D)
    a = {0: 1.0, 1: math.sqrt(5.0) / l, 2: math.sqrt(3.0) / l, 3: 1.0 / l}[kid]
    return J, sf2, l, a


def grad_params(kid, D, klam, rng) -> np.ndarray:
    """Hyper-parameters for the candidate-gradient cases: kernel_params' ranges with the length scales grown by sqrt(D / 3),
    so that distances in [0,1]^D stay of order one; SE-ARD with klam Lambda columns of entries N(0, 0.25 / D)."""
    s = 0.5 * math.log(max(D, 3) / 3.0)
    if kid == 0:
        return np.concatenate([rng.uniform(-0.7, 0.3, D) + s, rng.normal(0.0, 0.5 / math.sqrt(D), D * klam), [rng.uniform(-0.3, 0.3)]])
    return np.array([rng.uniform(-1.0, 0.0) + s, rng.uniform(-0.3, 0.3)])


def coef_lipschitz(kid, sf2, l, a):
    """(Lk, Lc): bounds of |dk/dd| and |dc/dd| over d >= 0, with k(d) the kernel value and c(d) the gradient coefficient
    (dk/du = c (u - u_n)) of oracle/acq_grad.kernel_and_coef:
      SE:   k = sf2 e^(-d^2/2),          c = -k:                     |k'|, |c'| <= sf2 d e^(-d^2/2) <= sf2
      Exp:  k = sf2 e^(-d^2/2l^2),       c = -k / l^2:               |k'| <= sf2 / l,  |c'| <= sf2 / l^3
      M5/2: k = sf2 (1 + ad + a^2d^2/3) e^(-ad), c = -sf2 a^2/3 (1 + ad) e^(-ad): |k'| = sf2 a (ad)(1 + ad)/3 e^(-ad) <= sf2 a,
            |c'| = sf2 a^3 (ad) e^(-ad) / 3 <= sf2 a^3
      M3/2: k = sf2 (1 + ad) e^(-ad),    c = -sf2 a^2 e^(-ad):      |k'| = sf2 a (ad) e^(-ad) <= sf2 a,  |c'| <= sf2 a^3"""
    if kid == 0:
        return sf2, sf2
    if kid == 3:
        return sf2 / l, sf2 / l ** 3
    return sf2 * a, sf2 * a ** 3


def _staged_pairs(kid, p, X, Xq):
    """Staged coordinates, the per-dimension differences q_e = u_e(candidate) - u_e(training point) (N x M each), the
    distances d and the kernel values k and coefficients c of every pair, in fp64."""
    from oracle import acq_grad as AG
    J, sf2, l, _ = staging(kid, p, X.shape[1])
    U_, Uq = X @ J, Xq @ J
    Q = [Uq[None, :, e] - U_[:, e, None] for e in range(J.shape[1])]
    z = np.zeros_like(Q[0])
    for q in Q:
        z += q * q
    k, c = AG.kernel_and_coef(kid, z, sf2, l)
    return J, U_, Uq, Q, np.sqrt(z), k, c


def grad_reference_ld(kid, p, X, Xq, L, alpha):
    """The same quantities as QueryCase.grad_reference (mu, sigma^2, grad mu of output 0, grad sigma^2), in np.longdouble
    throughout: staging, kernel values and coefficients, and both triangular solves by substitution.  For the host check
    that the fp64 reference stays inside the bounds below."""
    ld = np.longdouble
    X, Xq, p = X.astype(ld), Xq.astype(ld), np.asarray(p).astype(ld)
    D = X.shape[1]
    if kid == 0:
        klam = (p.size - 1 - D) // D
        J = np.hstack([np.diag(np.exp(-p[:D])), p[D:D + D * klam].reshape(klam, D).T])
        sf2, l = np.exp(2 * p[-1]), ld(1)
    else:
        J, sf2, l = np.eye(D, dtype=ld), np.exp(2 * p[1]), np.exp(p[0])
    U_, Uq = X @ J, Xq @ J
    Q = [Uq[None, :, e] - U_[:, e, None] for e in range(J.shape[1])]
    z = sum(q * q for q in Q)
    d = np.sqrt(z)
    if kid == 0:
        k = sf2 * np.exp(-z / 2)
        c = -k
    elif kid == 3:
        k = sf2 * np.exp(-z / (2 * l * l))
        c = -k / (l * l)
    elif kid == 1:
        a = np.sqrt(ld(5)) / l
        e = np.exp(-a * d)
        k, c = sf2 * (1 + a * d + a * a * z / 3) * e, -sf2 * (a * a / 3) * (1 + a * d) * e
    else:
        a = np.sqrt(ld(3)) / l
        e = np.exp(-a * d)
        k, c = sf2 * (1 + a * d) * e, -sf2 * a * a * e
    Lq = L.astype(ld)
    n, m = k.shape
    V = np.zeros((n, m), dtype=ld)
    for i in range(n):
        V[i] = (k[i] - Lq[i, :i] @ V[:i]) / Lq[i, i]
    W = np.zeros((n, m), dtype=ld)
    for i in range(n - 1, -1, -1):
        W[i] = (V[i] - Lq[i + 1:, i] @ W[i + 1:]) / Lq[i, i]
    a0 = alpha[:, 0].astype(ld)
    gmu = np.stack([(c * q).T @ a0 for q in Q], axis=1) @ J.T
    gs2 = np.stack([-2 * ((c * q) * W).sum(0) for q in Q], axis=1) @ J.T
    mu = k.T @ alpha.astype(ld)
    s2 = sf2 - (V * V).sum(0)
    return mu, s2, gmu, gs2


def grad_bounds(kid, p, X, Xq, alpha, noise, normE, ref):
    """First-order bounds on |x^ - x| for mu, sigma^2, grad mu (output 0) and grad sigma^2 of ONE fp64 evaluation (the
    device's or the host reference's: a comparison of the two uses twice these), per candidate (and dimension).  In staged
    coordinates u = x J, for each pair of a candidate and a training point n:
      staging:  |du_e| <= gamma_{D+3} (|x| |J|)_e per point (the reciprocal 1/ell, the Lambda dot product; 0 when J = I),
                |dq_ne| <= du_e(candidate) + du_e(n) + u |q_ne|;
      distance: |dd_n| <= ||dq_n||_2 + gamma_{De+6} d_n (the sum of De squares, the reciprocal square root);
      k and c:  |dk_n| <= Lk |dd_n| + gamma_16 (1 + rho_n) |k_n|, likewise c with Lc (coef_lipschitz), rho_n the exponent
                (exp < 3 ulp, its argument rho u, the polynomial and products < 8 roundings);
      solves:   ||dV_c|| <= kap^2 gamma_N ||V_c|| + ||L^-1|| ||dK*_c||,  ||dW_c|| <= kap^2 gamma_N ||W_c|| + ||L^-1|| ||dV_c||
                (bound_s2's forward bound, applied to L and then to L^T; kap = (1 + |E|)/(1 - |E|), ||L^-1|| <= 1/(c(1 - |E|)));
      sums:     gamma_{N+2} times the sum of |products| (two products, then N terms in any order: the device's per-thread
                chains, lane and warp trees; the host's BLAS);
      map:      g_x = J g_u with gamma_{De+3} |J| |g_u| (the products, the sum, and the rounding of J itself).
    ref: QueryCase.grad_reference's dict."""
    N, D = X.shape
    J, sf2, l, a = staging(kid, p, D)
    De = J.shape[1]
    aJ = np.abs(J)
    ident = kid != 0
    eu_x = np.zeros((N, De)) if ident else gamma(D + 3) * (np.abs(X) @ aJ)
    eu_q = np.zeros((Xq.shape[0], De)) if ident else gamma(D + 3) * (np.abs(Xq) @ aJ)
    Q, d, k, cc = ref["Q"], ref["d"], ref["Ks"], ref["c"]
    dQ = [eu_q[None, :, e] + eu_x[:, e, None] + U * np.abs(Q[e]) for e in range(De)]
    dd = np.sqrt(sum(x * x for x in dQ)) + gamma(De + 6) * d
    rho = {0: 0.5 * d * d, 3: 0.5 * (d / l) ** 2}.get(kid, a * d)
    Lk, Lc = coef_lipschitz(kid, sf2, l, a)
    g16 = gamma(16) * (1.0 + rho)
    dk = Lk * dd + g16 * np.abs(k)
    dc = Lc * dd + g16 * np.abs(cc)
    c = float(ref["L"][0, 0])
    kap = (1.0 + normE) / (1.0 - normE)
    nli = 1.0 / (c * (1.0 - normE))
    V, W = ref["V"], ref["W"]
    nv, nw = np.linalg.norm(V, axis=0), np.linalg.norm(W, axis=0)
    dV = kap * kap * gamma(N) * nv + nli * np.linalg.norm(dk, axis=0)
    dW = kap * kap * gamma(N) * nw + nli * dV
    a0 = np.abs(alpha[:, 0])[:, None]
    aW = np.abs(W)
    gN = gamma(N + 2)
    bmu_u, bs2_u, gu_mu, gu_s2 = [], [], [], []
    for e in range(De):
        aq, acq = np.abs(Q[e]), np.abs(cc * Q[e])
        pert = np.abs(cc) * dQ[e] + aq * dc
        bmu_u.append((a0 * pert).sum(0) + gN * (a0 * acq).sum(0))
        bs2_u.append(2.0 * ((aW * pert).sum(0) + gN * (aW * acq).sum(0) + np.linalg.norm(acq, axis=0) * dW))
        gu_mu.append(np.abs((cc * Q[e]).T @ alpha[:, 0]))
        gu_s2.append(np.abs(2.0 * ((cc * Q[e]) * W).sum(0)))
    bmu_u, bs2_u = np.stack(bmu_u, 1), np.stack(bs2_u, 1)
    gu_mu, gu_s2 = np.stack(gu_mu, 1), np.stack(gu_s2, 1)
    gJ = gamma(De + 3)
    v2 = nv * nv
    aal = np.abs(alpha)
    return dict(
        mu=gN * (np.abs(k).T @ aal) + dk.T @ aal,
        s2=2.0 * nv * dV + gN * v2 + 2.0 * U * (sf2 + v2 + abs(noise)),
        dmu=bmu_u @ aJ.T + gJ * (gu_mu @ aJ.T),
        ds2=bs2_u @ aJ.T + gJ * (gu_s2 @ aJ.T))


def bound_acq(acq_id, params, mu0, s2, dmu, ds2):
    """(value bound, gradient bound) of the UCB / EI epilogue evaluated in fp64 from given mu (output 0 plus the mean),
    sigma^2, grad mu and grad sigma^2, on the device and on the host (oracle/acq_grad.ucb / ei) together.
      UCB: v = mu + a sigma, g = grad mu + a grad s2 / (2 sigma): 4 roundings each side on |mu| + |a sigma| and on
           |grad mu| + |a grad s2 / 2 sigma|.
      EI:  X = mu - f - j (|dX| <= 2u(|mu| + |f| + |j|)), Z = X / sigma (|dZ| <= |dX| / sigma + 3u |Z|), Phi = erfc(-Z/sqrt2)/2
           (erfc <= 5 ulp on either side, plus phi |dZ| + u phi |Z| from its argument), phi = exp(-Z^2/2)/sqrt(2 pi)
           (phi (|Z| |dZ| + 6u)); g = Phi grad mu + phi grad s2 / (2 sigma) with 4 more roundings per term; the value
           X Phi + sigma phi likewise."""
    mu0, s2 = np.asarray(mu0), np.asarray(s2)
    sg = np.sqrt(s2)
    if acq_id == 0:
        aa = params[0]
        t = np.abs(aa * ds2 / (2.0 * sg)[:, None])
        return 2 * 4.0 * U * (np.abs(mu0) + np.abs(aa) * sg), 2 * 4.0 * U * (np.abs(dmu) + t)
    f, j = params
    from scipy.special import erfc
    Xv = mu0 - f - j
    Z = Xv / sg
    phi = np.exp(-0.5 * Z * Z) / math.sqrt(2.0 * math.pi)
    Phi = 0.5 * erfc(-Z / math.sqrt(2.0))
    dX = 2.0 * U * (np.abs(mu0) + abs(f) + abs(j))
    dZ = dX / sg + 3.0 * U * np.abs(Z)
    dPhi = 10.0 * U * Phi + phi * dZ + U * phi * np.abs(Z)
    dphi = phi * (np.abs(Z) * dZ + 6.0 * U)
    t = np.abs(ds2 / (2.0 * sg)[:, None])
    bg = dPhi[:, None] * np.abs(dmu) + dphi[:, None] * t + 2 * 4.0 * U * (Phi[:, None] * np.abs(dmu) + phi[:, None] * t)
    bv = np.abs(Xv) * dPhi + Phi * dX + sg * dphi + 2 * 4.0 * U * (np.abs(Xv) * Phi + sg * phi)
    return bv, bg


# ---------------------------------------------------------------------------------------------------------------------
# the device side (C ABI, include/limbo_b200.h)
# ---------------------------------------------------------------------------------------------------------------------
class Handle:
    """One lb_gp handle on device 0."""

    def __init__(self, lib, precision: int = 0):
        import ctypes as C
        from limbo_b200 import _lib
        self.C, self._lib, self.lib = C, _lib, lib
        lib.lb_debug_force_unfused_query.argtypes = [C.c_void_p, C.c_int]
        lib.lb_debug_force_unfused_query.restype = C.c_int
        self.h = C.c_void_p()
        _lib.check(lib.lb_create(C.byref(self.h), 0, precision), "lb_create")

    def close(self):
        if self.h:
            self.lib.lb_destroy(self.h)
            self.h = None

    def set_data(self, X, Y):
        X = np.ascontiguousarray(X, dtype=np.float64)
        Y = np.asfortranarray(Y, dtype=np.float64)
        self.N, self.D, self.P = X.shape[0], X.shape[1], Y.shape[1]
        self._keep = (X, Y)
        self._lib.check(self.lib.lb_set_data(self.h, self.N, self.D, self.P, X.ctypes.data, Y.ctypes.data), "lb_set_data")

    def set_kernel(self, kid, p, noise):
        p = np.ascontiguousarray(p, dtype=np.float64)
        self._lib.check(self.lib.lb_set_kernel(self.h, kid, p.ctypes.data, p.size, float(noise)), "lb_set_kernel")
        self.nh = p.size

    def load_factor(self, L, alpha):
        L = np.asfortranarray(L, dtype=np.float64)
        alpha = np.asfortranarray(alpha, dtype=np.float64)
        self._lib.check(self.lib.lb_load_factor(self.h, L.ctypes.data, alpha.ctypes.data), "lb_load_factor")

    def fit(self):
        self._lib.check(self.lib.lb_fit(self.h), "lb_fit")

    def factor(self, K) -> int:
        """Factor K in place of the stored factor: lb_load_factor puts K (and the identity in the padding) where lb_fit's
        kernel build would, lb_stage_potrf factors it and rebuilds the diagonal-block inverses, lb_check_info returns
        dpotrf's info.  Returns that info (0 or the 1-based failing pivot)."""
        self.load_factor(K, np.zeros((self.N, self.P)))
        self._lib.check(self.lib.lb_stage_potrf(self.h), "lb_stage_potrf")
        rc = int(self.lib.lb_check_info(self.h))
        if rc < 0:
            self._lib.check(rc, "lb_check_info")
        return rc

    def refit_alpha(self, Y):
        Y = np.asfortranarray(Y, dtype=np.float64)
        self._lib.check(self.lib.lb_refit_alpha(self.h, Y.ctypes.data), "lb_refit_alpha")

    def get(self, what):
        n = self.N
        out = np.empty((n, self.P) if what == 2 else (n, n), order="F")
        self._lib.check(self.lib.lb_get(self.h, what, out.ctypes.data), "lb_get")
        return out

    def log_lik(self) -> float:
        v = self.C.c_double()
        self._lib.check(self.lib.lb_log_lik(self.h, self.C.addressof(v)), "lb_log_lik")
        return v.value

    def grad(self, optimize_noise: bool):
        g = np.empty(self.nh + (1 if optimize_noise else 0))
        self._lib.check(self.lib.lb_kernel_grad_log_lik(self.h, int(optimize_noise), g.ctypes.data), "lb_kernel_grad_log_lik")
        return g

    def query(self, Xq, unfused: bool = False):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        mu = np.empty((M, self.P))
        s2 = np.empty(M)
        self.lib.lb_debug_force_unfused_query(self.h, int(unfused))
        try:
            self._lib.check(self.lib.lb_query(self.h, M, Xq.ctypes.data, mu.ctypes.data, s2.ctypes.data), "lb_query")
        finally:
            self.lib.lb_debug_force_unfused_query(self.h, 0)
        return mu, s2

    def query_grad(self, Xq):
        """lb_query_grad: mu (M x P), sigma^2, grad mu and grad sigma^2 (M x D)."""
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        mu, s2, dmu, ds2 = np.empty((M, self.P)), np.empty(M), np.empty((M, self.D)), np.empty((M, self.D))
        self._lib.check(self.lib.lb_query_grad(self.h, M, Xq.ctypes.data, mu.ctypes.data, s2.ctypes.data, dmu.ctypes.data,
                                               ds2.ctypes.data), "lb_query_grad")
        return mu, s2, dmu, ds2

    def acq_grad(self, acq_id, params, Xq, mean=None, mean_const=0.0, mean_grad=None):
        """lb_acq_grad: the acquisition's values and gradients (M, M x D)."""
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        ap = np.array(list(params) + [0.0] * (2 - len(params)), dtype=np.float64)
        mean = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        mean_grad = None if mean_grad is None else np.ascontiguousarray(mean_grad, dtype=np.float64)
        v, g = np.empty(M), np.empty((M, self.D))
        self._lib.check(self.lib.lb_acq_grad(self.h, acq_id, ap.ctypes.data, M, Xq.ctypes.data,
                                             None if mean is None else mean.ctypes.data, float(mean_const),
                                             None if mean_grad is None else mean_grad.ctypes.data, v.ctypes.data, g.ctypes.data),
                        "lb_acq_grad")
        return v, g

    def acq_argmax(self, acq_id, params, Xq, mean=None, mean_const=0.0):
        """lb_acq_argmax: (values, best value, best index)."""
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        ap = np.array(list(params) + [0.0] * (2 - len(params)), dtype=np.float64)
        mean = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        v, best, idx = np.empty(M), self.C.c_double(), self.C.c_int64()
        self._lib.check(self.lib.lb_acq_argmax(self.h, acq_id, ap.ctypes.data, M, Xq.ctypes.data,
                                               None if mean is None else mean.ctypes.data, float(mean_const), v.ctypes.data,
                                               self.C.addressof(best), self.C.addressof(idx)), "lb_acq_argmax")
        return v, best.value, idx.value


def factor_outputs(h: Handle, case: ExactCase, X) -> dict:
    """L, alpha and K^-1 of an exact case on handle h (data, kernel, factor, alpha)."""
    h.set_data(X, case.Y)
    h.set_kernel(0, np.zeros(X.shape[1] + 1), 0.01)
    info = h.factor(case.K)
    assert info == 0, info
    h.refit_alpha(case.Y)
    return dict(L=h.get(1), alpha=h.get(2), kinv=h.get(3))
