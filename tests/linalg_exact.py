"""Matrices with an exactly known Cholesky factor, numpy restatements of the kernel derivatives (SE-ARD with its Lambda
columns included), and first-order rounding-error bounds for the fp64 factorisation, inverse, solves and query, the
likelihood and LOO-CV objectives and their gradients, K^-1 obs_mean, and the batched likelihood of a K built from X
(tests/test_linalg_exact_host.py, tests/test_gpu_linalg_exact.py, tests/test_gpu_objectives_exact.py).

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



EXACT_KLAM = (0, 1, 2, 4)


def exact_objective(i: int, N: int):
    """(kernel id, D, Lambda columns, optimize_noise) of the i-th exact shape: the kernels cycle through the four, SE-ARD
    carries k = 0, 1, 2, 4 Lambda columns in turn, the noise entry alternates, and D = 20 at N = 1151 (two 16-dimension passes
    of the gradient kernels, and dk_build's loop over 24 staged dimensions)."""
    kid = KERNELS[i % 4]
    klam = EXACT_KLAM[(i // 4) % 4] if kid == 0 else 0
    D = 20 if (kid == 0 and N == 1151) else 2
    return kid, D, klam, bool((i // 4) % 2)


def exact_objective_params(kid, D, klam, rng) -> np.ndarray:
    """kernel_params, with the D = 20 case's longer length scales (ell in e^[0.3, 0.8], sigma_f = e^0.1)."""
    if D == 20:
        lam = rng.normal(0.0, 0.5 / math.sqrt(D), D * klam) if klam else np.zeros(0)
        return np.concatenate([rng.uniform(0.3, 0.8, D), lam, [0.1]])
    return kernel_params(kid, D, rng, klam)

# ---------------------------------------------------------------------------------------------------------------------
# kernels: values and derivatives (the formulas of oracle/limbo_oracle.hpp, vectorised)
# ---------------------------------------------------------------------------------------------------------------------
def kernel_params(kid: int, D: int, rng, klam: int = 0) -> np.ndarray:
    """Log-space hyper-parameters; SE-ARD with klam Lambda columns of entries N(0, 0.25 / D) (A(i, j) = p[(j + 1) D + i])."""
    if kid == 0:
        ell = rng.uniform(-0.7, 0.3, D)
        lam = rng.normal(0.0, 0.5 / math.sqrt(D), D * klam) if klam else np.zeros(0)
        return np.concatenate([ell, lam, [rng.uniform(-0.3, 0.3)]])
    return np.array([rng.uniform(-1.0, 0.0), rng.uniform(-0.3, 0.3)])


def ard_split(p, D):
    """SE-ARD's (klam, 1/ell, Lambda (D x klam), sf2) from its log-space parameters, in p's dtype."""
    klam = (p.size - 1 - D) // D
    assert p.size == D + D * klam + 1, (p.size, D)
    return klam, np.exp(-p[:D]), p[D:D + D * klam].reshape(klam, D).T, np.exp(2 * p[-1])


def _sqdist(X1, X2, scale=None):
    """Squared distances from the coordinate differences (no Gram-matrix trick, which cancels for close points)."""
    A = X1 if scale is None else X1 * scale
    B = X2 if scale is None else X2 * scale
    z = np.zeros((X1.shape[0], X2.shape[0]), dtype=A.dtype)
    for d in range(A.shape[1]):
        q = A[:, d, None] - B[None, :, d]
        z += q * q
    return z


def _ard_z(p, X1, X2):
    """SE-ARD's squared distance in the staged coordinates [x / ell, x^T Lambda] and its parts."""
    klam, inv, A, sf2 = ard_split(p, X1.shape[1])
    z = _sqdist(X1, X2, inv)
    U1, U2 = X1 @ A, X2 @ A
    if klam:
        z = z + _sqdist(U1, U2)
    return z, inv, U1, U2, sf2


def kernel_matrix(kid: int, p: np.ndarray, X1: np.ndarray, X2: np.ndarray) -> np.ndarray:
    """k(x1, x2) without noise, as in Kernel::kernel of each functor (in the inputs' dtype)."""
    c = X1.dtype.type
    if kid == 0:
        z, _, _, _, sf2 = _ard_z(p, X1, X2)
        return sf2 * np.exp(-z / 2)
    l, sf2 = np.exp(p[0]), np.exp(2 * p[1])
    s = _sqdist(X1, X2)
    if kid == 3:
        return sf2 * np.exp(-s / (2 * l * l))
    r = np.sqrt(s)
    if kid == 1:
        t1 = np.sqrt(c(5)) * r / l
        t2 = 5 * s / (3 * l * l)
        return sf2 * (1 + t1 + t2) * np.exp(-t1)
    t = np.sqrt(c(3)) * r / l
    return sf2 * (1 + t) * np.exp(-t)


def kernel_grads(kid: int, p: np.ndarray, X1: np.ndarray, X2: np.ndarray):
    """Yields dk(x1, x2) / d theta_q for every hyper-parameter q as matrices, in the order of the functor's parameters: SE-ARD
    log ell_d, then Lambda entry A(i, j) at q = (j + 1) D + i (squared_exp_ard.hpp:119-122: -k (x1 - x2)^T A(:, j) (x1 - x2)_i),
    then log sigma_f; the isotropic kernels log l, then log sigma_f.  In the inputs' dtype (long double for the host checks)."""
    c = X1.dtype.type
    if kid == 0:
        D = X1.shape[1]
        z, inv, U1, U2, sf2 = _ard_z(p, X1, X2)
        k = sf2 * np.exp(-z / 2)
        for d in range(D):
            q = (X1[:, d, None] - X2[None, :, d]) * inv[d]
            yield q * q * k
        for j in range(U1.shape[1]):
            proj = U1[:, j, None] - U2[None, :, j]
            for i in range(D):
                yield -(proj * (X1[:, i, None] - X2[None, :, i])) * k
        yield 2 * k
        return
    l, sf2 = np.exp(p[0]), np.exp(2 * p[1])
    s = _sqdist(X1, X2)
    if kid == 3:
        r = s / (l * l)
        k = sf2 * np.exp(-r / 2)
        yield r * k
        yield 2 * k
        return
    d = np.sqrt(s)
    if kid == 1:
        t1 = np.sqrt(c(5)) * d / l
        t2 = 5 * s / (3 * l * l)
        e = np.exp(-t1)
        yield sf2 * (e * t1 * (1 + t1 + t2) + (-t1 - 2 * t2) * e)
        yield 2 * sf2 * (1 + t1 + t2) * e
        return
    t = np.sqrt(c(3)) * d / l
    e = np.exp(-t)
    yield sf2 * (-t * e + (1 + t) * t * e)
    yield 2 * sf2 * (1 + t) * e


def kernel_eval_err(kid: int, p: np.ndarray, xmax: float, D: int) -> float:
    """Absolute bound on the fp64 evaluation error of one kernel value or derivative, inputs in [-xmax, xmax]^D.
    Every formula is sf^2 * (polynomial of degree <= 3 in rho) * exp(-rho) of the squared distance z, Lipschitz in z
    with constant <= sf^2 (1 + a^2)(1 + rho)^2 (a: the scale of z inside rho); z itself is a sum of De squared differences
    of staged coordinates u = x J, so |dz| <= gamma_{D+3} zb with zb the largest sum over e of (2 xmax sum_d |J_de|)^2.
    SE-ARD's Lambda entries -k proj raw (proj = (x1 - x2)^T A(:, j), raw = (x1 - x2)_i, |proj| <= sqrt(zb), |raw| <= 2 xmax)
    add sf^2 (|d proj| |raw| + |proj| |d raw| + |proj raw| |dk| / sf^2) <= sf^2 2 xmax sqrt(zb) (2 + zb) gamma_{D+3}."""
    lam = 0.0
    if kid == 0:
        klam, inv, A, sf2 = ard_split(np.asarray(p, dtype=np.float64), D)
        J = np.hstack([np.diag(inv), A])
        zb = float(((2.0 * xmax * np.abs(J).sum(0)) ** 2).sum())
        a2, rho = 1.0, 0.5 * zb
        if klam:
            lam = sf2 * 2.0 * xmax * math.sqrt(zb) * (2.0 + zb) * gamma(D + 3)
    else:
        l, sf2 = math.exp(p[0]), math.exp(2 * p[1])
        zb = D * (2.0 * xmax) ** 2
        if kid == 3:
            a2 = 1.0 / (l * l)
            rho = 0.5 * a2 * zb
        else:
            a2 = (5.0 if kid == 1 else 3.0) / (l * l)
            rho = math.sqrt(a2 * zb)
    return sf2 * ((1.0 + a2) * (1.0 + rho) ** 2 * gamma(D + 3) * zb + gamma(32) * (1.0 + rho) ** 3 * (1.0 + zb)) + lam


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


def dk_matrices(kid, p, X, noise, optimize_noise):
    """dK / d theta_q for every hyper-parameter (kernel_grads), then 2 noise I when the noise is optimised (kernel.hpp:90-93)."""
    out = list(kernel_grads(kid, p, X, X))
    if optimize_noise:
        out.append(2 * noise * np.eye(X.shape[0], dtype=X.dtype))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# leave-one-out cross-validation (gp.hpp:339-399) and K^-1 obs_mean (gp.hpp:313-330)
# ---------------------------------------------------------------------------------------------------------------------
def loo_value(alpha, kinv) -> float:
    """sum_i,p -1/2 alpha_ip^2 / c_i - 1/2 log(1 / c_i) - 1/2 log(2 pi), c = diag(K^-1) (gp.hpp:339-351)."""
    ic = 1 / np.diag(kinv)
    dt = ic.dtype.type
    return (-alpha * alpha * ic[:, None] / 2 - np.log(ic)[:, None] / 2 - np.log(2 * dt(np.pi)) / 2).sum()


def loo_terms(alpha, kinv, dk, cols=None):
    """(alpha Z alpha - 1/2 (1 + alpha^2 / c) diag(Z K^-1)) / c per row and output, Z = K^-1 dK (gp.hpp:353-399); cols: the
    columns n of Z alpha and of diag(Z K^-1) = sum_n Z_in K^-1_ni to sum (the device's 128-column tiles), all by default."""
    ic = 1 / np.diag(kinv)
    Z = kinv @ dk
    if cols is None:
        za, zk = Z @ alpha, (Z * kinv).sum(1)
    else:
        za, zk = Z[:, cols] @ alpha[cols], (Z[:, cols] * kinv[:, cols]).sum(1)
    return Z, za, zk, (alpha * za - (1 + alpha * alpha * ic[:, None]) * zk[:, None] / 2) * ic[:, None]


def loo_reference(kid, p, X, alpha, kinv, noise, optimize_noise):
    """LOO value and gradient in the dtype of the inputs (np.longdouble for the host checks)."""
    g = [loo_terms(alpha, kinv, dk)[3].sum() for dk in dk_matrices(kid, p, X, noise, optimize_noise)]
    return loo_value(alpha, kinv), np.array(g)


def bound_loo(case: ExactCase, da_bound, dkinv_bound) -> float:
    """|v^ - v| for the LOO value from K^-1 and alpha with ||d alpha_p|| <= da_bound[p] and ||dK^-1||_F <= dkinv_bound
    (device and reference together): the derivatives -alpha / c (alpha) and 1/2 (alpha^2 / c^2 + 1 / c) (c_i = K^-1_ii) by
    Cauchy-Schwarz, then the terms (a division, a log, four products and sums: 10 roundings each) and the sum of N P of them,
    on the device and on the host."""
    kinv, a = case.ref()["kinv"], case.A0
    ic = 1.0 / np.diag(kinv)
    w = 0.5 * (a * a * (ic * ic)[:, None] + ic[:, None]).sum(1)
    first = float((np.linalg.norm(a * ic[:, None], axis=0) * da_bound).sum() + np.linalg.norm(w) * dkinv_bound)
    terms = float((0.5 * a * a * ic[:, None] + 0.5 * np.abs(np.log(ic))[:, None] + 0.5 * math.log(2 * math.pi)).sum())
    return first + 2.0 * gamma(case.N * case.P + 10) * terms


def bound_loo_grad(case: ExactCase, kid, p, X, noise, optimize_noise, da_bound, dkinv_bound) -> np.ndarray:
    """|g^ - g| per hyper-parameter of the LOO gradient, from K^-1 (X, ||dX||_F <= dkinv_bound), alpha (a, ||da_p|| <=
    da_bound[p]) and dK (evaluation error ev per entry, kernel_eval_err; the noise entry's 2 noise I is exact), first order:
      alpha:    t_ip = (a Za - 1/2 (1 + a^2/c) zk) / c moves by ic (da Za + a (Z da) - a da ic zk): by ||.||_2 per output;
      X in Z:   Za by dX dK a (sum_ip |a ic| |dX dK a| <= ||a ic|| ||dX|| ||dK a||), zk = diag(X dK X) by (dX M)_ii + (M^T dX)_ii
                with M = dK X: sum_i v_i ||dX_i,:|| ||M_:,i|| <= ||dX||_F ||v ||M_:,i|| ||, twice (v_i = sum_p (1 + a^2 ic) ic / 2);
      c = diag(X): d t / d c_i = (-a Za + zk / 2 + a^2 zk ic) ic^2, by ||.||_2;
      Z product (DMMA on the device, BLAS on the host): |dZ| <= gamma_N |X||dK| = gamma_N G; the epilogue's sums over the N
                columns (per 128-column tile, then over the T tiles) add gamma_{N+T} |Z||a| <= G|a| and |Z||X| <= G|X|:
                |dZa| <= 2 gamma_{N+T+2} G|a|, |dzk_i| <= 2 gamma_{N+T+2} (G|X|)_ii;
      ev:       |dZa_ip| <= ev (|X| 1)_i sum |a_p|, |dzk_i| <= ev (|X| 1)_i^2;
      the terms and the final sum: gamma_{NP+10} sum |t|.
    The rounding and evaluation terms are counted twice (device and host)."""
    n, P = case.N, case.P
    Xk, a = case.ref()["kinv"], case.A0
    ic = 1.0 / np.diag(Xk)
    absX = np.abs(Xk)
    r1 = absX.sum(1)
    v = 0.5 * ((1.0 + a * a * ic[:, None]) * ic[:, None]).sum(1)
    T = max(1, -(-n // TILE))
    gz = gamma(n + T + 2)
    ev = kernel_eval_err(kid, p, float(np.abs(X).max()), X.shape[1])
    dks = dk_matrices(kid, p, X, noise, optimize_noise)
    out = []
    for q, dk in enumerate(dks):
        is_noise = optimize_noise and q == len(dks) - 1
        Z, za, zk, t = loo_terms(a, Xk, dk)
        aic = a * ic[:, None]
        b = 0.0
        for pp in range(P):
            b += da_bound[pp] * (np.linalg.norm(ic * za[:, pp]) + np.linalg.norm(Z.T @ aic[:, pp])
                                 + np.linalg.norm(ic * ic * a[:, pp] * zk))
        M = dk @ Xk
        b += dkinv_bound * (float(np.linalg.norm(aic, axis=0) @ np.linalg.norm(dk @ a, axis=0))
                            + 2.0 * np.linalg.norm(v * np.linalg.norm(M, axis=0)))
        s = ((-a * za + 0.5 * zk[:, None] + a * a * zk[:, None] * ic[:, None]) * (ic * ic)[:, None]).sum(1)
        b += dkinv_bound * np.linalg.norm(s)
        G = absX @ np.abs(dk)
        rnd = float((np.abs(aic) * (2.0 * gz * (G @ np.abs(a)))).sum() + (v * 2.0 * gz * (G * absX).sum(1)).sum())
        evt = 0.0 if is_noise else ev * float((np.abs(aic) * (r1[:, None] * np.abs(a).sum(0)[None, :])).sum() + (v * r1 * r1).sum())
        fin = gamma(n * P + 10) * float((np.abs(a * za * ic[:, None]) + 0.5 * (1.0 + a * a * ic[:, None]) * np.abs(zk)[:, None]
                                         * ic[:, None]).sum())
        out.append(b + 2.0 * (rnd + evt + fin))
    return np.array(out)


def bound_kinv_obs(case: ExactCase, dkinv_bound) -> np.ndarray:
    """2-norm bound per column on (K^-1 Y)^ - A0 (Y = K A0 exactly): ||dX||_2 ||y_p|| from the K^-1 bound, and the dot products
    over 32 slices of N and the sum of the 32 partials, gamma_{N+32} || |X| |y_p| ||_2."""
    Xk, Y = case.ref()["kinv"], case.Y
    return dkinv_bound * np.linalg.norm(Y, axis=0) + gamma(case.N + 32) * np.linalg.norm(np.abs(Xk) @ np.abs(Y), axis=0)


# ---------------------------------------------------------------------------------------------------------------------
# the log-likelihood and its gradient of a K built from X (lb_lml_grad_batch)
# ---------------------------------------------------------------------------------------------------------------------
JITTER = 1e-8  # kernel.hpp:83, on the diagonal of every K


class LmlCase:
    """GP::compute_log_lik and compute_kernel_grad_log_lik (gp.hpp:267-311) at one kernel state, in fp64 through LAPACK, with
    the quantities of its first-order bound (bound())."""

    def __init__(self, kid, p, noise, X, Y, optimize_noise):
        import scipy.linalg as sl
        self.kid, self.p, self.noise, self.X, self.Y, self.on = kid, np.asarray(p, dtype=np.float64), noise, X, Y, optimize_noise
        n = X.shape[0]
        K = kernel_matrix(kid, self.p, X, X)
        K[np.diag_indices(n)] += noise + JITTER
        ev = sl.eigh(K, eigvals_only=True)
        self.K, self.lmin, self.lmax = K, float(ev[0]), float(ev[-1])
        self.kappa = self.lmax / self.lmin
        L = np.linalg.cholesky(K)
        self.L = L
        self.alpha = sl.cho_solve((L, True), Y)
        Li = sl.solve_triangular(L, np.eye(n), lower=True)
        self.kinv = Li.T @ Li
        self.logdet = 2.0 * float(np.log(np.diag(L)).sum())
        ya = float((Y * self.alpha).sum())
        self.lik = -0.5 * ya - 0.5 * self.logdet - 0.5 * n * math.log(2 * math.pi)
        self.grad, self.absum, self.fro = grad_reference(kid, self.p, X, self.alpha, self.kinv, noise, optimize_noise)

    def bound(self):
        """(likelihood bound, gradient bound per entry) of ONE fp64 evaluation from X (the device's or this reference's):
          K:        |dK_ij| <= ev (kernel_eval_err) and 2u K_ii on the diagonal (noise and jitter added): ||dK_b||_F;
          factor:   backward error gamma_{3N+1} || |L||L^T| ||_F of the Cholesky factorisation and both solves (Thm 10.3/10.4),
                    added to dK_b: dK;
          alpha:    ||d alpha_p|| <= ||K^-1||_2 dK ||alpha_p||;  K^-1: ||dX||_F <= ||K^-1||_2^2 dK sqrt(N) (section 14.2);
          log det:  |tr(K^-1 dK)| <= ||K^-1||_F dK, and gamma_{N+4} sum |2 log L_ii| for the logs and their sum;
          y^T alpha: sum_p ||y_p|| ||d alpha_p|| + gamma_{NP+2} sum |y||alpha|; the likelihood's three terms: 4 roundings;
          gradient: bound_grad's terms from d alpha and dX, ev sum |W| / 2 and gamma_{N^2+P+8} sum |W||dk|."""
        n = self.X.shape[0]
        ev = kernel_eval_err(self.kid, self.p, float(np.abs(self.X).max()), self.X.shape[1])
        absL = np.abs(self.L)
        dKb = math.sqrt(n * (n - 1)) * ev + math.sqrt(n) * (ev + 2.0 * U * float(np.diag(self.K).max()))
        dK = dKb + gamma(3 * n + 1) * float(np.linalg.norm(absL @ absL.T))
        nki = 1.0 / self.lmin
        da = nki * dK * np.linalg.norm(self.alpha, axis=0)
        dX = nki * nki * dK * math.sqrt(n)
        dld = math.sqrt(n) * nki * dK + gamma(n + 4) * float(np.abs(2.0 * np.log(np.diag(self.L))).sum())
        ya = float((self.Y * self.alpha).sum())
        dya = float((np.linalg.norm(self.Y, axis=0) * da).sum()) + gamma(n * self.Y.shape[1] + 2) * float(np.abs(self.Y * self.alpha).sum())
        blik = 0.5 * (dya + dld) + gamma(4) * (0.5 * abs(ya) + 0.5 * abs(self.logdet) + 0.5 * n * math.log(2 * math.pi))
        W = self.alpha @ self.alpha.T - self.kinv
        dW = float(2.0 * (da * np.linalg.norm(self.alpha, axis=0)).sum() + dX)
        bgrad = 0.5 * dW * self.fro + 2.0 * gamma(n * n + self.Y.shape[1] + 8) * self.absum + 0.5 * ev * float(np.abs(W).sum())
        return blik, bgrad


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


    def loo_cv(self) -> float:
        v = self.C.c_double()
        self._lib.check(self.lib.lb_log_loo_cv(self.h, self.C.addressof(v)), "lb_log_loo_cv")
        return v.value

    def loo_grad(self, optimize_noise: bool):
        g = np.empty(self.nh + (1 if optimize_noise else 0))
        self._lib.check(self.lib.lb_kernel_grad_log_loo_cv(self.h, int(optimize_noise), g.ctypes.data), "lb_kernel_grad_log_loo_cv")
        return g

    def kinv_obs(self):
        """lb_kinv_obs_mean: K^-1 obs_mean (N x P)."""
        out = np.empty((self.N, self.P), order="F")
        self._lib.check(self.lib.lb_kinv_obs_mean(self.h, out.ctypes.data), "lb_kinv_obs_mean")
        return out

    def append(self, x, Yall):
        """lb_append: one sample x (D) and the refreshed (N + 1) x P obs_mean."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        Yall = np.asfortranarray(Yall, dtype=np.float64)
        self._lib.check(self.lib.lb_append(self.h, x.ctypes.data, Yall.ctypes.data), "lb_append")
        self.N += 1
        self._keep = (self._keep[0], Yall)

    def lml_grad_batch(self, kid, H, noise, optimize_noise: bool):
        """lb_lml_grad_batch at the rows of H (R x n_hparams) and noise (R): (lik, grad, info)."""
        H = np.ascontiguousarray(H, dtype=np.float64)
        noise = np.ascontiguousarray(noise, dtype=np.float64)
        R, nh = H.shape
        lik, grad = np.empty(R), np.empty((R, nh + (1 if optimize_noise else 0)))
        info = np.empty(R, dtype=np.int32)
        self._lib.check(self.lib.lb_lml_grad_batch(self.h, kid, R, nh, H.ctypes.data, noise.ctypes.data, int(optimize_noise),
                                                   lik.ctypes.data, grad.ctypes.data, info.ctypes.data), "lb_lml_grad_batch")
        return lik, grad, info

def factor_outputs(h: Handle, case: ExactCase, X) -> dict:
    """L, alpha and K^-1 of an exact case on handle h (data, kernel, factor, alpha)."""
    h.set_data(X, case.Y)
    h.set_kernel(0, np.zeros(X.shape[1] + 1), 0.01)
    info = h.factor(case.K)
    assert info == 0, info
    h.refit_alpha(case.Y)
    return dict(L=h.get(1), alpha=h.get(2), kinv=h.get(3))
