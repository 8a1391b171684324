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
