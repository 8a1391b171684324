"""Host checks of the exact-factor harness (tests/linalg_exact.py): the constructed K, Y and truths are exact, every
case is well conditioned, the vectorised kernel derivatives match the oracle, and the bounds hold for LAPACK."""
import math

import numpy as np
import pytest
import scipy.linalg as sl

import linalg_exact as E


@pytest.mark.parametrize("N,P,seed", [(1, 1, 1), (255, 3, 2), (1153, 5, 3)])
def test_case_is_exact(N, P, seed):
    c = E.ExactCase(N, P, seed)
    Li = c.L0.astype(np.int64)
    Ki = Li @ Li.T  # integer arithmetic: exact
    assert np.abs(Ki).max() < 2 ** 53
    assert np.array_equal(c.K, Ki.astype(np.float64))
    Ai = np.rint(c.A0 / E.A0_SCALE).astype(np.int64)
    assert np.array_equal(Ai.astype(np.float64) * E.A0_SCALE, c.A0)
    assert np.array_equal(c.Y, (Ki @ Ai).astype(np.float64) * E.A0_SCALE)
    d = np.diag(c.L0)
    assert np.all((d >= 2 ** 11) & (d <= 2 ** 12)) and np.abs(np.tril(c.L0, -1)).max(initial=0) <= 8
    ld = 2 * np.sum(np.log(d.astype(np.longdouble)))
    assert abs(c.logdet - float(ld)) <= 4 * E.U * abs(c.logdet)
    # LAPACK's factor of K is L0 to rounding
    Lc = np.linalg.cholesky(c.K)
    assert np.linalg.norm(Lc - c.L0) <= E.bound_L(c)


@pytest.mark.parametrize("N,P,seed", E.exact_shapes(), ids=[f"N{n}" for n, _, _ in E.exact_shapes()])
def test_kappa_of_every_case(N, P, seed):
    c = E.ExactCase(N, P, seed)
    r = c.ref()
    assert 1.0 <= r["kappa"] < 16.0, r["kappa"]
    assert r["c_blk"] < 8.0, r["c_blk"]
    print(f"N={N} kappa_2(K)={r['kappa']:.3f} c_blk={r['c_blk']:.3f}")


@pytest.mark.parametrize("N,seed", [(64, 5), (700, 6), (2049, 7)])
def test_bounds_hold_for_lapack(N, seed):
    """The reference pipeline (LAPACK dpotrf, dpotrs, numpy inverse) stays inside every bound; a perturbed factor
    (one 128 x 128 tile scaled by 1 + 2^-30) does not."""
    c = E.ExactCase(N, 3, seed)
    Lc = np.linalg.cholesky(c.K)
    eL, bL = np.linalg.norm(Lc - c.L0), E.bound_L(c)
    a = sl.cho_solve((Lc, True), c.Y)
    ea, ba = np.linalg.norm(a - c.A0, axis=0), E.bound_alpha(c)
    ki = np.linalg.inv(c.K)
    ek, bk = np.linalg.norm(ki - c.ref()["kinv"]), E.bound_kinv(c)
    ld = 2 * np.sum(np.log(np.diag(Lc)))
    print(f"N={N} ratios L={eL / bL:.2e} alpha={np.max(ea / ba):.2e} Kinv={ek / bk:.2e}")
    assert eL <= bL and np.all(ea <= ba) and ek <= bk
    assert abs(ld - c.logdet) <= E.bound_logdet(c)
    # a one-tile value perturbation of the factor exceeds the bound
    Lp = Lc.copy()
    t0 = max(0, (N - 1) // 128 * 128)
    Lp[t0:, t0:t0 + 128] *= 1.0 + 2.0 ** -30
    assert np.linalg.norm(Lp - c.L0) > bL


def test_bad_pivot_matches_dpotrf():
    c = E.ExactCase(700, 1, 9)
    for p in (0, 31, 32, 127, 128, 255, 256, 511, 512, 699):
        Kb = c.with_bad_pivot(p)
        _, info = sl.lapack.dpotrf(Kb, lower=1)
        assert info == p + 1, (p, info)
        # the Schur complement at p is exactly -K_pp / 2
        r = math.fsum(float(v) ** 2 for v in c.L0[p, :p])
        assert Kb[p, p] - r == -0.5 * c.K[p, p]


def test_gamma():
    assert E.gamma(1) == pytest.approx(E.U, rel=1e-15)
    assert E.gamma(2 ** 20) > 2 ** 20 * E.U
    with pytest.raises(AssertionError):
        E.gamma(2 ** 53)


@pytest.mark.parametrize("kid", E.KERNELS, ids=[E.KERNEL_NAMES[k] for k in E.KERNELS])
@pytest.mark.parametrize("D", [1, 3, 20])
def test_vectorised_kernel_and_derivatives_match_oracle(oracle_mod, kid, D):
    O = oracle_mod
    rng = np.random.default_rng(100 + 10 * kid + D)
    p = E.kernel_params(kid, D, rng)
    X1 = rng.uniform(0.0, 1.0, size=(6, D))
    X2 = np.vstack([X1[:2], rng.uniform(0.0, 1.0, size=(5, D))])  # includes zero distances
    K = E.kernel_matrix(kid, p, X1, X2)
    G = list(E.kernel_grads(kid, p, X1, X2))
    assert len(G) == p.size
    ev = E.kernel_eval_err(kid, p, 1.0, D)
    for i in range(X1.shape[0]):
        for j in range(X2.shape[0]):
            k_o = O.kernel_eval(kid, p, 0.0, X1[i], X2[j])
            g_o = O.kernel_grad(kid, p, X1[i], X2[j])
            assert abs(K[i, j] - k_o) <= 2 * ev, (i, j, K[i, j], k_o)
            for q in range(p.size):
                assert abs(G[q][i, j] - g_o[q]) <= 2 * ev, (i, j, q, G[q][i, j], g_o[q])


@pytest.mark.parametrize("kid", E.KERNELS, ids=[E.KERNEL_NAMES[k] for k in E.KERNELS])
@pytest.mark.parametrize("optimize_noise", [False, True])
def test_gradient_formula_matches_oracle_gp(oracle_mod, kid, optimize_noise):
    """0.5 sum_ij (alpha alpha^T - K^-1)_ij dk_ij against OracleGP.grad on small kernel-matrix problems."""
    O = oracle_mod
    rng = np.random.default_rng(200 + kid)
    for N, D, P in [(5, 1, 1), (40, 3, 2), (130, 20 if kid == 0 else 2, 1)]:
        X = rng.uniform(0.0, 1.0, size=(N, D))
        Y = rng.normal(size=(N, P))
        p = E.kernel_params(kid, D, rng)
        og = O.OracleGP()
        og.set_data(X, Y)
        og.set_kernel(kid, p, 0.01)
        assert og.fit() == -1  # the restated Cholesky returns -1 when every pivot is positive
        alpha, kinv = og.get(2), og.get(3)
        g, absum, _ = E.grad_reference(kid, p, X, alpha, kinv, 0.01, optimize_noise)
        go = og.grad(optimize_noise)
        assert np.all(np.abs(g - go) <= 1e-12 * (absum + np.abs(go).max())), (N, g, go)


def test_query_case_conditioning():
    qc = E.QueryCase(300, 3, 2, 5)
    assert qc.norm_E() <= 0.25
    A = np.eye(300) + qc.E
    assert np.linalg.cond(A) <= 5.0 / 3.0
    p = E.kernel_params(1, 3, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(50, 3))
    L, mu, s2, V, Ks = qc.reference(1, p, 0.01, Xq)
    sf2 = math.exp(2 * p[-1])
    assert (V * V).sum(0).max() == pytest.approx(sf2 / 2, rel=1e-12)
    assert np.all(s2 - 0.01 >= sf2 / 2 * (1 - 1e-12))
    # the bounds cover an independent evaluation (numpy solve of L, not of I + E)
    V2 = np.linalg.solve(L, Ks)
    s2b = sf2 - (V2 * V2).sum(0) + 0.01
    bs = E.bound_s2(1, p, V, float(L[0, 0]), qc.norm_E(), 1.0, 3, 0.01)
    assert np.all(np.abs(s2b - s2) <= bs)
    bm = E.bound_mu(1, p, Ks, qc.alpha, 1.0, 3)
    mu2 = np.einsum("ij,ip->jp", Ks, qc.alpha)
    assert np.all(np.abs(mu2 - mu) <= bm)


# ---- candidate gradients on a loaded factor ----------------------------------------------------------------------------
GRAD_CASES = [(0, 3, 0), (0, 3, 2), (1, 3, 0), (2, 3, 0), (3, 3, 0), (0, 17, 1), (1, 17, 0)]


def _grad_case(kid, D, klam, N, M, seed, P=2):
    qc = E.QueryCase(N, D, P, seed)
    p = E.grad_params(kid, D, klam, qc.rng)
    Xq = qc.rng.uniform(0.0, 1.0, size=(M, D))
    return qc, p, Xq


@pytest.mark.parametrize("kid,D,klam", GRAD_CASES)
def test_grad_reference_central_differences(kid, D, klam):
    """The reference's gradients against central differences of its own mu (output 0) and sigma^2, the factor fixed."""
    qc, p, Xq = _grad_case(kid, D, klam, 200, 12, 300 + 10 * kid + klam)
    r = qc.grad_reference(kid, p, 0.01, Xq)
    H = 1e-5
    scale = np.maximum(np.abs(np.hstack([r["dmu"], r["ds2"]])).max(axis=1), 1e-3)
    for d in range(D):
        e = np.zeros(D)
        e[d] = H
        rp, rm = qc.grad_reference(kid, p, 0.01, Xq + e, L=r["L"]), qc.grad_reference(kid, p, 0.01, Xq - e, L=r["L"])
        fd_mu = (rp["mu"][:, 0] - rm["mu"][:, 0]) / (2 * H)
        fd_s2 = (rp["s2"] - rm["s2"]) / (2 * H)
        assert np.all(np.abs(r["dmu"][:, d] - fd_mu) <= 1e-6 * scale), np.abs(r["dmu"][:, d] - fd_mu).max()
        assert np.all(np.abs(r["ds2"][:, d] - fd_s2) <= 1e-6 * scale), np.abs(r["ds2"][:, d] - fd_s2).max()


@pytest.mark.parametrize("kid,D,klam", GRAD_CASES)
def test_grad_reference_matches_oracle_formulas(kid, D, klam):
    """oracle/acq_grad.query_grad (K^-1 K* by cho_solve, differences in one M x N x De array) on the same L, within twice
    the one-evaluation bounds."""
    from oracle import acq_grad as AG
    qc, p, Xq = _grad_case(kid, D, klam, 300, 40, 400 + 10 * kid + klam)
    r = qc.grad_reference(kid, p, 0.01, Xq)
    b = E.grad_bounds(kid, p, qc.X, Xq, qc.alpha, 0.01, qc.norm_E(), r)
    mu, s2, dmu, ds2, _ = AG.query_grad(kid, p, 0.01, qc.X, r["L"], qc.alpha, Xq)
    for name, got in (("mu", mu), ("s2", s2), ("dmu", dmu), ("ds2", ds2)):
        ratio = float(np.max(np.abs(got - r[name]) / (2.0 * b[name])))
        print(f"kid={kid} D={D} klam={klam} {name} ratio={ratio:.2e}")
        assert ratio <= 1.0, name


@pytest.mark.parametrize("kid,D,klam,N", [(1, 3, 0, 127), (2, 3, 0, 2049), (3, 16, 0, 300), (0, 15, 2, 1000), (0, 3, 0, 4224),
                                          (1, 3, 0, 4224)])
def test_grad_bounds_hold_for_scipy(kid, D, klam, N):
    """SciPy's fp64 gradients stay inside the one-evaluation bounds against a long-double substitution reference; scaling
    W's last 128-row tile by 1 + 2^-30 (the size of a one-tile slip of the backward walk) leaves them."""
    qc, p, Xq = _grad_case(kid, D, klam, N, 6, 500 + N + kid)
    r = qc.grad_reference(kid, p, 0.01, Xq)
    b = E.grad_bounds(kid, p, qc.X, Xq, qc.alpha, 0.01, qc.norm_E(), r)
    mu, s2, dmu, ds2 = E.grad_reference_ld(kid, p, qc.X, Xq, r["L"], qc.alpha)
    s2 = s2 + 0.01
    ratios = {}
    for name, ref in (("mu", mu), ("s2", s2), ("dmu", dmu), ("ds2", ds2)):
        err = np.abs(r[name] - ref).astype(np.float64)
        ratios[name] = float(np.max(err / b[name]))
    print(f"kid={kid} D={D} klam={klam} N={N} ratios", {k: f"{v:.2e}" for k, v in ratios.items()})
    assert all(v <= 1.0 for v in ratios.values()), ratios
    # a perturbation the size of the last super-block's 2^-30 slip exceeds the bound
    W = r["W"].copy()
    t0 = (N - 1) // 128 * 128
    W[t0:] *= 1.0 + 2.0 ** -30
    J = E.staging(kid, p, D)[0]
    ds2p = np.stack([-2.0 * ((r["c"] * q) * W).sum(0) for q in r["Q"]], axis=1) @ J.T
    assert float(np.max(np.abs(ds2p - ds2).astype(np.float64) / b["ds2"])) > 1.0


def test_acq_bounds_hold_for_long_double():
    """bound_acq covers the UCB / EI epilogue of oracle/acq_grad against the same formulas in long double."""
    from oracle import acq_grad as AG
    rng = np.random.default_rng(600)
    M, D = 400, 3
    mu0 = rng.normal(size=M)
    s2 = np.exp(rng.uniform(-4.0, 1.0, M))
    dmu, ds2 = rng.normal(size=(M, D)), rng.normal(size=(M, D)) * s2[:, None]
    for acq_id, params in ((0, [0.6]), (1, [0.4, 0.01]), (1, [3.0, 0.0])):
        v, g = AG.ucb(mu0, s2, dmu, ds2, params[0]) if acq_id == 0 else AG.ei(mu0, s2, dmu, ds2, *params)
        bv, bg = E.bound_acq(acq_id, params, mu0, s2, dmu, ds2)
        ld = np.longdouble
        sg = np.sqrt(s2.astype(ld))
        if acq_id == 0:
            rv = mu0 + ld(params[0]) * sg
            rg = dmu + ld(params[0]) * ds2 / (2 * sg)[:, None]
        else:
            import mpmath
            Xv = mu0.astype(ld) - ld(params[0]) - ld(params[1])
            Z = Xv / sg
            with mpmath.workdps(30):
                Phi = np.array([ld(str(mpmath.ncdf(mpmath.mpf(str(z))))) for z in Z], dtype=ld)
            phi = np.exp(-Z * Z / 2) / np.sqrt(2 * ld(np.pi))
            rv = Xv * Phi + sg * phi
            rg = Phi[:, None] * dmu + phi[:, None] * ds2 / (2 * sg)[:, None]
        rv_, rg_ = float(np.max(np.abs(v - rv).astype(np.float64) / bv)), float(np.max(np.abs(g - rg).astype(np.float64) / bg))
        print(f"acq={acq_id} {params} ratio value={rv_:.2e} grad={rg_:.2e}")
        assert rv_ <= 1.0 and rg_ <= 1.0


# ---- SE-ARD Lambda columns, LOO-CV, K^-1 obs_mean and the batched likelihood ------------------------------------------
@pytest.mark.parametrize("klam", [1, 2, 4])
@pytest.mark.parametrize("D", [1, 3, 20])
def test_lambda_derivatives_match_oracle(oracle_mod, D, klam):
    """SE-ARD with klam Lambda columns (A(i, j) at (j + 1) D + i): kernel_matrix against the oracle's K, and the likelihood
    gradient built from every kernel_grads entry against OracleGP.grad, which sums the functor's own gradient
    (squared_exp_ard.hpp:119-122) over the pairs."""
    O = oracle_mod
    rng = np.random.default_rng(700 + 10 * D + klam)
    for N, P in [(7, 1), (60, 2)]:
        p = E.kernel_params(0, D, rng, klam)
        assert p.size == D * (1 + klam) + 1
        X = rng.uniform(0.0, 1.0, size=(N, D))
        Y = rng.normal(size=(N, P))
        og = O.OracleGP()
        og.set_data(X, Y)
        og.set_kernel(0, p, 0.01)
        assert og.fit() == -1
        K = E.kernel_matrix(0, p, X, X)
        K[np.diag_indices(N)] += 0.01 + E.JITTER
        ev = E.kernel_eval_err(0, p, 1.0, D)
        assert np.abs(K - og.get(0)).max() <= 2 * ev + 4 * E.U
        G = list(E.kernel_grads(0, p, X, X))
        assert len(G) == p.size
        for q in range(D, p.size - 2):  # neighbouring Lambda slots differ (a slot written one entry off would show)
            assert np.abs(G[q] - G[q + 1]).max() > 2 * ev, q
        alpha, kinv = og.get(2), og.get(3)
        g, absum, _ = E.grad_reference(0, p, X, alpha, kinv, 0.01, True)
        go = og.grad(True)
        assert np.all(np.abs(g - go) <= 1e-12 * (absum + np.abs(go).max())), (N, g, go)


@pytest.mark.parametrize("kid,klam", [(0, 0), (0, 2), (1, 0), (2, 0), (3, 0)])
def test_loo_formula_matches_oracle_gp(oracle_mod, kid, klam):
    """loo_reference (value and gradient, noise optimised) against OracleGP.loo_cv / loo_grad on kernel-matrix problems."""
    O = oracle_mod
    rng = np.random.default_rng(800 + 10 * kid + klam)
    for N, D, P in [(5, 1, 1), (40, 3, 2), (130, 3, 1)]:
        X = rng.uniform(0.0, 1.0, size=(N, D))
        Y = rng.normal(size=(N, P))
        p = E.kernel_params(kid, D, rng, klam)
        og = O.OracleGP()
        og.set_data(X, Y)
        og.set_kernel(kid, p, 0.01)
        assert og.fit() == -1
        v, g = E.loo_reference(kid, p, X, og.get(2), og.get(3), 0.01, True)
        vo, go = og.loo_cv(), og.loo_grad(True)
        assert abs(v - vo) <= 1e-10 * abs(vo), (N, v, vo)
        assert np.all(np.abs(g - go) <= 1e-9 * np.abs(go).max()), (N, g, go)


def _inv_lower_ld(L):
    """L^-1 of a lower-triangular matrix by substitution in long double."""
    n = L.shape[0]
    Lq = L.astype(np.longdouble)
    Li = np.zeros((n, n), dtype=np.longdouble)
    for i in range(n):
        Li[i, i] = 1 / Lq[i, i]
        Li[i, :i] = -(Lq[i, :i] @ Li[:i, :i]) / Lq[i, i]
    return Li


def _tiles(N):
    return [slice(t, min(t + 128, N)) for t in range(0, N, 128)]


LOO_CASES = [(127, 1, 0, 2, True), (130, 3, 1, 0, False), (256, 5, 0, 4, True), (300, 2, 3, 0, True)]


@pytest.mark.parametrize("N,P,kid,klam,on", LOO_CASES)
def test_loo_and_kinv_obs_bounds_hold_for_long_double(N, P, kid, klam, on):
    """The fp64 LOO value and gradient (LAPACK K^-1 of the exact factor, alpha = A0) and K^-1 Y stay inside bound_loo,
    bound_loo_grad and bound_kinv_obs against the same formulas in long double.  Scaling the value's rows of any one
    128-row tile by 1 + 2^-30 leaves its bound; dropping any one tile's contribution to K^-1 Y (the K^-1 bound grows as N^2 u
    and is of the order of a 2^-30 slip there from N = 256 on), or its partials of Z alpha and diag(Z K^-1) from the gradient (its bound carries the evaluation error of dK, kernel_eval_err's
    worst case over the whole input box, which is far above the rounding of the products)."""
    c = E.ExactCase(N, P, 1200 + N)
    rng = np.random.default_rng(N)
    X = rng.uniform(0.0, 1.0, size=(N, 2))
    p = E.kernel_params(kid, 2, rng, klam)
    noise = 0.01
    kinv = c.ref()["kinv"]
    ba, bk = E.bound_alpha(c), E.bound_kinv(c)
    v64, g64 = E.loo_reference(kid, p, X, c.A0, kinv, noise, on)
    Li = _inv_lower_ld(c.L0)
    kld = Li.T @ Li
    ld = np.longdouble
    vld, gld = E.loo_reference(kid, p.astype(ld), X.astype(ld), c.A0.astype(ld), kld, ld(noise), on)
    bv, bg = E.bound_loo(c, ba, bk), E.bound_loo_grad(c, kid, p, X, noise, on, ba, bk)
    rv, rg = float(abs(v64 - vld) / bv), np.abs(g64 - gld).astype(np.float64) / bg
    ko64 = kinv @ c.Y
    bko = E.bound_kinv_obs(c, bk)
    rko = np.linalg.norm(ko64 - c.A0, axis=0) / bko
    print(f"N={N} kid={kid} klam={klam} ratios loo={rv:.2e} loo_grad={rg.max():.2e} kinv_obs={rko.max():.2e}")
    assert rv <= 1.0 and np.all(rg <= 1.0) and np.all(rko <= 1.0)
    # one tile's contribution scaled by 1 + 2^-30 (value) or dropped (K^-1 Y, gradient) exceeds the bound, for every tile
    eps = 2.0 ** -30
    ic = 1.0 / np.diag(kinv)
    rows = -c.A0 * c.A0 * ic[:, None] / 2 - np.log(ic)[:, None] / 2 - math.log(2 * math.pi) / 2
    dks = E.dk_matrices(kid, p, X, noise, on)
    for t in _tiles(N):
        assert abs(eps * rows[t].sum()) > bv, ("value", t)
        assert np.all(np.linalg.norm(kinv[:, t] @ c.Y[t], axis=0) > bko), ("kinv_obs", t)
        gt = np.array([E.loo_terms(c.A0, kinv, dk, t)[3].sum() for dk in dks])
        assert np.all(np.abs(gt) > bg), ("grad", t, np.abs(gt) / bg)


def _chol_ld(K):
    n = K.shape[0]
    L = np.zeros_like(K)
    for j in range(n):
        d = K[j, j] - L[j, :j] @ L[j, :j]
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (K[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def lml_ld(case: E.LmlCase):
    """The likelihood and gradient of an LmlCase in long double throughout (kernel, Cholesky, solves, inverse, gradient)."""
    ld = np.longdouble
    X, p, Y = case.X.astype(ld), case.p.astype(ld), case.Y.astype(ld)
    n = X.shape[0]
    K = E.kernel_matrix(case.kid, p, X, X)
    K[np.diag_indices(n)] += ld(case.noise) + ld(E.JITTER)
    L = _chol_ld(K)
    Li = _inv_lower_ld(L)
    kinv = Li.T @ Li
    alpha = kinv @ Y
    lik = -(Y * alpha).sum() / 2 - np.log(np.diag(L)).sum() - n * np.log(2 * ld(np.pi)) / 2
    W = alpha @ alpha.T - kinv
    g = [(W * dk).sum() / 2 for dk in E.dk_matrices(case.kid, p, X, ld(case.noise), case.on)]
    return lik, np.array(g)


GCH = 8  # lml_batch.cu: SE-ARD ell / Lambda gradient entries per sweep


@pytest.mark.parametrize("kid,N,D,klam,P,on", [(0, 33, 3, 2, 2, True), (0, 128, 4, 4, 1, False), (1, 200, 3, 0, 2, True),
                                               (3, 127, 5, 0, 1, True)])
def test_lml_bounds_hold_for_long_double(kid, N, D, klam, P, on):
    """LmlCase's fp64 likelihood and gradient stay inside its bound against long double, kappa_2(K) <= 1e4; for SE-ARD,
    swapping two neighbouring ell / Lambda entries (across the first GCH sweep boundary and the ell / Lambda boundary) or
    dropping the last sweep's entries exceeds twice the bound (the device-against-reference bar)."""
    rng = np.random.default_rng(1300 + N)
    X = rng.uniform(0.0, 1.0, size=(N, D))
    Y = rng.normal(size=(N, P))
    p = E.grad_params(kid, D, klam, rng)
    noise = lml_noise(p, N)
    c = E.LmlCase(kid, p, noise, X, Y, on)
    assert c.kappa <= 1e4, c.kappa
    bl, bg = c.bound()
    lik, g = lml_ld(c)
    rl, rg = float(abs(c.lik - lik) / bl), np.abs(c.grad - g).astype(np.float64) / bg
    print(f"kid={kid} N={N} kappa={c.kappa:.1f} ratios lik={rl:.2e} grad={rg.max():.2e}")
    assert rl <= 1.0 and np.all(rg <= 1.0)
    if kid == 0:
        nent = D * (1 + klam)
        for a_, b_ in {(D - 1, D), (GCH - 1, GCH)}:
            if b_ < nent:
                gs = c.grad.copy()
                gs[[a_, b_]] = gs[[b_, a_]]
                assert np.any(np.abs(gs - c.grad) > 2 * bg), ("swap", a_, b_)
        last = (nent - 1) // GCH * GCH
        assert np.any(np.abs(c.grad[last:nent]) > 2 * bg[last:nent]), "drop the last sweep"


def lml_noise(p, N):
    """A noise that keeps kappa_2(K) <= 1e4: lambda_max <= N sf2 + noise, lambda_min >= noise."""
    return 0.01 + N * math.exp(2 * p[-1]) / 8000.0
