"""Candidate gradients on the device (lb_query_grad / lb_acq_grad): against the NumPy / SciPy formulas of oracle/acq_grad.py, against
lb_query / lb_acq_argmax bit for bit on the panel path, against central differences of the device's own lb_query, the edge cases
(clamp, EI cut-off, no samples), determinism and batch independence, plumbing (leases, launches, errors), and the gradient
acquisition optimiser bayes_opt.BatchedGradientSearch."""
import ctypes as C
import gc
import math

import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky
from scipy.optimize import minimize
from scipy.spatial.distance import cdist

from dropin import run_dropin
from oracle import acq_grad as AG

pytestmark = pytest.mark.gpu

LB_ERR_ARG, LB_ERR_UNSUPPORTED = -1, -5
CASES = [(AG.K_SE_ARD, 0), (AG.K_SE_ARD, 2), (AG.K_MATERN52, 0), (AG.K_MATERN32, 0), (AG.K_EXP, 0)]
TOL = 1e-9  # of the per-candidate magnitude sum_n |g_n| (|alpha_n0| + 2 |W_nc|)


def _lib():
    from limbo_b200 import _lib as L
    return L, L.load()


def _p(a):
    return a.ctypes.data if a is not None else None


class _Handle:
    def __init__(self, kid, X, Y, hp, noise, precision=0):
        self.L, self.lib = _lib()
        self.h = C.c_void_p()
        self.L.check(self.lib.lb_create(C.byref(self.h), 0, precision), "lb_create")
        X = np.ascontiguousarray(X, dtype=np.float64)
        Y = np.asfortranarray(Y, dtype=np.float64)
        self.D, self.P = X.shape[1], Y.shape[1]
        self.L.check(self.lib.lb_set_data(self.h, X.shape[0], self.D, self.P, _p(X) if X.size else None, _p(Y) if Y.size else None), "set_data")
        hp = np.ascontiguousarray(hp, dtype=np.float64)
        self.L.check(self.lib.lb_set_kernel(self.h, kid, _p(hp), hp.size, noise), "set_kernel")
        if X.shape[0]:
            self.L.check(self.lib.lb_fit(self.h), "fit")

    def __del__(self):
        self.lib.lb_destroy(self.h)

    def query_grad(self, Xq):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        mu, s2, dmu, ds2 = np.empty((M, self.P)), np.empty(M), np.empty((M, self.D)), np.empty((M, self.D))
        self.L.check(self.lib.lb_query_grad(self.h, M, _p(Xq), _p(mu), _p(s2), _p(dmu), _p(ds2)), "lb_query_grad")
        return mu, s2, dmu, ds2

    def acq_grad(self, acq_id, params, Xq):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        ap = np.array(list(params) + [0.0] * (2 - len(params)), dtype=np.float64)
        v, g = np.empty(M), np.empty((M, self.D))
        self.L.check(self.lib.lb_acq_grad(self.h, acq_id, _p(ap), M, _p(Xq), None, 0.0, None, _p(v), _p(g)), "lb_acq_grad")
        return v, g

    def query(self, Xq):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        mu, s2 = np.empty((M, self.P)), np.empty(M)
        self.L.check(self.lib.lb_query(self.h, M, _p(Xq), _p(mu), _p(s2)), "lb_query")
        return mu, s2

    def acq_values(self, acq_id, params, Xq):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        M = Xq.shape[0]
        ap = np.array(list(params) + [0.0] * (2 - len(params)), dtype=np.float64)
        v, best, idx = np.empty(M), C.c_double(), C.c_int64()
        self.L.check(self.lib.lb_acq_argmax(self.h, acq_id, _p(ap), M, _p(Xq), None, 0.0, _p(v), C.addressof(best), C.addressof(idx)),
                     "lb_acq_argmax")
        return v


def _problem(kid, klam, N, D=3, P=2, seed=0, log_sf=0.0, noise=0.01):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    Y = np.stack([np.sin(3 * X[:, 0]) + X[:, -1] ** 2, np.cos(2 * X[:, 1])], axis=1)[:, :P]
    Y = Y - Y.mean(axis=0)
    hp = np.concatenate([np.log(rng.uniform(0.3, 0.8, D)), 0.6 * rng.standard_normal(D * klam), [log_sf]]) if kid == AG.K_SE_ARD \
        else np.array([math.log(0.4), log_sf])
    return X, Y, hp, noise


def _reference(kid, hp, noise, X, Y, Xq):
    """oracle/acq_grad.py over K = k(X, X) + (noise + 1e-8) I (kernel.hpp:83), its SciPy factor and alpha"""
    J, sf2, l = AG.staging(kid, hp, X.shape[1])
    U = X @ J
    K, _ = AG.kernel_and_coef(kid, cdist(U, U, "sqeuclidean"), sf2, l)
    K[np.diag_indices_from(K)] += noise + 1e-8
    L = cholesky(K, lower=True)
    return AG.query_grad(kid, hp, noise, X, L, cho_solve((L, True), Y), Xq)


@pytest.mark.parametrize("N", [1, 127, 300, 2100, 4500])
@pytest.mark.parametrize("kid,klam", CASES)
def test_against_the_numpy_formulas(kid, klam, N):
    X, Y, hp, noise = _problem(kid, klam, N)
    h = _Handle(kid, X, Y, hp, noise)
    rng = np.random.default_rng(N + 7)
    f_max = 0.3
    worst = 0.0
    for M in (1, 100, 300):
        Xq = rng.random((M, 3))
        mu, s2, dmu, ds2 = h.query_grad(Xq)
        rmu, rs2, rdmu, rds2, mag = _reference(kid, hp, noise, X, Y, Xq)
        assert np.allclose(mu, rmu, rtol=0, atol=1e-10) and np.allclose(s2, rs2, rtol=0, atol=1e-10)
        scale = mag + 1e-300
        for a, b in ((dmu, rdmu), (ds2, rds2)):
            r = np.abs(a - b) / scale
            worst = max(worst, float(r.max()))
            assert np.all(np.abs(a - b) <= TOL * scale + 1e-15), r.max()
        for acq_id, params, fun in ((0, [0.6], lambda: AG.ucb(rmu[:, 0], rs2, rdmu, rds2, 0.6)),
                                    (1, [f_max, 0.01], lambda: AG.ei(rmu[:, 0], rs2, rdmu, rds2, f_max, 0.01))):
            v, g = h.acq_grad(acq_id, params, Xq)
            rv, rg = fun()
            assert np.allclose(v, rv, rtol=0, atol=1e-10)
            assert np.all(np.abs(g - rg) <= 4 * TOL * scale + 1e-15)
    print(f"ACQGRAD_ERR kid={kid} klam={klam} N={N} max|err|/magnitude={worst:.3e}")


@pytest.mark.parametrize("kid,klam", CASES)
def test_values_equal_the_value_paths(kid, klam):
    from limbo_b200 import _lib as L
    lib = L.load()
    X, Y, hp, noise = _problem(kid, klam, 700)
    h = _Handle(kid, X, Y, hp, noise)
    rng = np.random.default_rng(3)
    for M in (300, 40, 1):
        Xq = rng.random((M, 3))
        mu, s2, _, _ = h.query_grad(Xq)
        for acq_id, params in ((0, [0.6]), (1, [0.2, 0.01])):
            v, _ = h.acq_grad(acq_id, params, Xq)
            if M >= 256:  # the panel path: bit for bit
                mq, sq = h.query(Xq)
                assert np.array_equal(mu, mq) and np.array_equal(s2, sq)
                assert np.array_equal(v, h.acq_values(acq_id, params, Xq))
            else:  # the slab / one-point paths: within 1e-12; with the panel threshold lowered, bit for bit
                mq, sq = h.query(Xq)
                assert np.allclose(mu, mq, rtol=0, atol=1e-12) and np.allclose(s2, sq, rtol=0, atol=1e-12)
                assert np.allclose(v, h.acq_values(acq_id, params, Xq), rtol=0, atol=1e-12)
                lib.lb_debug_set_query_panel_min(1)
                try:
                    if M > 1:  # lb_query of one point always takes the one-point kernel
                        mq, sq = h.query(Xq)
                        assert np.array_equal(mu, mq) and np.array_equal(s2, sq)
                    assert np.array_equal(v, h.acq_values(acq_id, params, Xq))
                finally:
                    lib.lb_debug_set_query_panel_min(0)


@pytest.mark.parametrize("kid,klam", CASES)
def test_central_differences_of_the_device(kid, klam):
    X, Y, hp, noise = _problem(kid, klam, 500)
    h = _Handle(kid, X, Y, hp, noise)
    Xq = np.random.default_rng(4).random((8, 3))
    _, _, dmu, ds2 = h.query_grad(Xq)
    H = 1e-5
    for d in range(3):
        e = np.zeros(3)
        e[d] = H
        (mp, sp), (mm, sm) = h.query(Xq + e), h.query(Xq - e)
        for an, fd in ((dmu[:, d], (mp[:, 0] - mm[:, 0]) / (2 * H)), (ds2[:, d], (sp - sm) / (2 * H))):
            scale = np.maximum(np.abs(np.stack([dmu, ds2])).max(axis=(0, 2)), 1e-3)
            assert np.all(np.abs(an - fd) <= 1e-6 * scale), np.abs(an - fd).max()


def test_clamp_and_ei_cutoff():
    """sigma_f^2 = e^-40 < DBL_EPSILON: the clamp is active everywhere; with noise 0, sigma = 0 < 1e-10 and EI is 0"""
    X, Y, hp, _ = _problem(AG.K_SE_ARD, 0, 200, log_sf=-20.0)
    h = _Handle(AG.K_SE_ARD, X, Y, hp, 0.0)
    Xq = np.vstack([X[:5], np.random.default_rng(5).random((300, 3))])
    mu, s2, dmu, ds2 = h.query_grad(Xq)
    assert np.all(s2 == 0.0) and np.all(ds2 == 0.0) and np.all(np.isfinite(dmu))
    v, g = h.acq_grad(1, [0.0, 0.0], Xq)
    assert np.all(v == 0.0) and np.all(g == 0.0)
    v, g = h.acq_grad(0, [0.5], Xq)
    assert np.array_equal(g, dmu)


def test_no_samples_gives_the_prior_and_a_zero_gradient():
    from limbo_b200 import kernel, model
    gp = model.GP(3, 1, kernel=kernel.MaternFiveHalves)
    Xq = np.random.default_rng(6).random((50, 3))
    mu, s2, dmu, ds2 = gp.query_grad_batch(Xq)
    mq, sq = gp.query_batch(Xq)
    assert np.array_equal(mu, mq) and np.array_equal(s2, sq)
    assert np.all(dmu == 0.0) and np.all(ds2 == 0.0)


def test_bits_do_not_depend_on_the_batch_or_the_call():
    X, Y, hp, noise = _problem(AG.K_MATERN52, 0, 2300)
    h = _Handle(AG.K_MATERN52, X, Y, hp, noise)
    rng = np.random.default_rng(8)
    Xq = rng.random((300, 3))
    a = h.query_grad(Xq)
    b = h.query_grad(Xq)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    perm = rng.permutation(300)
    c = h.query_grad(Xq[perm])
    assert all(np.array_equal(x[perm], y) for x, y in zip(a, c))
    pad = np.vstack([rng.random((77, 3)), Xq, rng.random((500, 3))])
    d = h.query_grad(pad)
    assert all(np.array_equal(x, y[77:377]) for x, y in zip(a, d))
    va, ga = h.acq_grad(1, [0.1, 0.0], Xq)
    vd, gd = h.acq_grad(1, [0.1, 0.0], pad)
    assert np.array_equal(va, vd[77:377]) and np.array_equal(ga, gd[77:377])


def _round(lib):
    from limbo_b200 import acqui, kernel, model
    rng = np.random.default_rng(9)
    X = rng.random((150, 2))
    gp = model.GP(2, 1, kernel=kernel.SquaredExpARD)
    gp.compute(X, np.sin(4 * X[:, :1]))
    Xq = rng.random((400, 2))
    gp.query_grad_batch(Xq)
    gp.acq_grad_batch(0, [0.5], Xq[:3])
    acqui.EI(gp).grad_batch(Xq)
    acqui.UCB(gp)(Xq[0], gradient=True)
    del gp


def test_round_returns_every_lease():
    L, lib = _lib()
    _round(lib)
    gc.collect()
    live = lib.lb_debug_pool_live()
    _round(lib)
    gc.collect()
    assert lib.lb_debug_pool_live() == live


def test_launch_count_does_not_grow_with_the_batch():
    X, Y, hp, noise = _problem(AG.K_EXP, 0, 3000)
    h = _Handle(AG.K_EXP, X, Y, hp, noise)
    rng = np.random.default_rng(10)
    h.query_grad(rng.random((10, 3)))  # the cached diagonal-block inverses are built on the first call
    counts = []
    for M in (1, 300, 3000):
        before = h.lib.lb_launch_count(h.h)
        h.acq_grad(0, [0.5], rng.random((M, 3)))
        counts.append(h.lib.lb_launch_count(h.h) - before)
    assert counts[0] == counts[1] == counts[2], counts


def test_errors():
    X, Y, hp, noise = _problem(AG.K_MATERN32, 0, 100)
    h = _Handle(AG.K_MATERN32, X, Y, hp, noise)
    lib = h.lib
    Xq = np.random.default_rng(11).random((4, 3))
    out = np.empty((4, 3))
    v = np.empty(4)
    ap = np.array([0.5, 0.0])
    assert lib.lb_query_grad(h.h, 0, _p(Xq), None, None, _p(out), None) == LB_ERR_ARG
    assert lib.lb_acq_grad(h.h, 0, _p(ap), 0, _p(Xq), None, 0.0, None, _p(v), _p(out)) == LB_ERR_ARG
    assert lib.lb_acq_grad(h.h, 7, _p(ap), 4, _p(Xq), None, 0.0, None, _p(v), _p(out)) == LB_ERR_ARG
    bad = Xq.copy()
    bad[2, 1] = np.nan
    assert lib.lb_query_grad(h.h, 4, _p(bad), None, None, _p(out), None) == LB_ERR_ARG
    assert lib.lb_acq_grad(h.h, 1, _p(ap), 4, _p(bad), None, 0.0, None, _p(v), _p(out)) == LB_ERR_ARG
    tf = _Handle(AG.K_MATERN32, X, Y, hp, noise, precision=1)
    assert lib.lb_query_grad(tf.h, 4, _p(Xq), None, None, _p(out), None) == LB_ERR_UNSUPPORTED
    assert lib.lb_acq_grad(tf.h, 0, _p(ap), 4, _p(Xq), None, 0.0, None, _p(v), _p(out)) == LB_ERR_UNSUPPORTED


class _OptParams:
    class acqui_ucb:
        alpha = 0.5

    class acqui_ei:
        jitter = 0.0

    class opt_batchedgradient:
        candidates = 2000
        starts = 16
        iterations = 300
        alpha = 0.01

    class opt_batchedrandom:
        candidates = 2000
        refinements = 2
        shrink = 0.1


@pytest.mark.parametrize("acq_name", ["UCB", "EI"])
@pytest.mark.parametrize("kname", ["SquaredExpARD", "MaternFiveHalves"])
def test_gradient_search_reaches_the_lbfgsb_maximum(kname, acq_name, oracle_mod):
    O = oracle_mod
    from limbo_b200 import acqui, bayes_opt, kernel, model
    rng = np.random.default_rng(12)
    X = rng.random((60, 2))
    y = np.sin(5 * X[:, :1]) * np.cos(3 * X[:, 1:]) + 0.3 * X[:, :1]
    gp = model.GP(2, 1, params=_OptParams, kernel=getattr(kernel, kname))
    gp.compute(X, y)
    acq = getattr(acqui, acq_name)(gp, 0, params=_OptParams)
    # the acquisition of the oracle's fit of the same data and h-params (mean::Data: the mean of y), with oracle/acq_grad.py's
    # gradients; f_max = max_i mu(x_i) over the oracle's own posterior mean (ei.hpp:100-108)
    kid = gp.kernel_function().kernel_id
    hp = np.asarray(gp.kernel_function().params(), dtype=np.float64)
    og = O.OracleGP()
    og.set_data(X, y - y.mean())
    og.set_kernel(kid, hp, gp.kernel_function().noise())
    og.fit()
    Lo, ao = og.get(1), og.get(2)
    f_max = float(og.query(X)[0][:, 0].max() + y.mean())

    def neg(x):
        mu, s2, dmu, ds2, _ = AG.query_grad(kid, hp, og.noise, X, Lo, ao, np.atleast_2d(x))
        mu0 = mu[:, 0] + y.mean()
        v, g = AG.ucb(mu0, s2, dmu, ds2, 0.5) if acq_name == "UCB" else AG.ei(mu0, s2, dmu, ds2, f_max, 0.0)
        return -float(v[0]), -g[0]
    starts = np.vstack([rng.random((40, 2)), np.stack(np.meshgrid(np.linspace(0.05, 0.95, 6), np.linspace(0.05, 0.95, 6)), -1).reshape(-1, 2)])
    best = max(-minimize(neg, s, jac=True, method="L-BFGS-B", bounds=[(0, 1), (0, 1)], options={"ftol": 1e-15, "gtol": 1e-12}).fun
               for s in starts)
    xg = bayes_opt.BatchedGradientSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    xr = bayes_opt.BatchedRandomSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    vg, vr = acq.grad_batch(np.vstack([xg, xr]))[0]
    assert vg >= best - 1e-6, (vg, best)
    assert vg >= vr


def test_boptimizer_runs_with_the_gradient_search():
    from limbo_b200 import acqui, bayes_opt, kernel, model, synth

    class P(_OptParams):
        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 10

        class opt_batchedgradient:
            candidates = 2000
            starts = 16
            iterations = 30
            alpha = 0.01
    gp = model.GP(6, 1, params=P, kernel=kernel.SquaredExpARD)
    bo = bayes_opt.BOptimizer(gp, params=P, acqui=acqui.UCB, acqui_opt=bayes_opt.BatchedGradientSearch(P, np.random.default_rng(1)),
                              rng=np.random.default_rng(1))
    bo.optimize(lambda x: synth.hartmann6(np.atleast_2d(x))[0], 6)
    assert len(bo.samples()) == 20
    assert all(np.all(np.isfinite(s)) and np.all((s >= 0) & (s <= 1)) for s in bo.samples())
    assert np.isfinite(bo.best_observation()[0])


def test_no_samples_acquisition_follows_the_mean():
    """the prior's acquisition on the device: UCB = mean + alpha sqrt(k(v, v) + noise), EI from the mean alone; the mean's
    input gradient passes through (times Phi(Z) for EI)"""
    L, lib = _lib()
    h = _Handle(AG.K_MATERN52, np.zeros((0, 2)), np.zeros((0, 1)), np.array([math.log(0.4), 0.0]), 0.01)
    rng = np.random.default_rng(13)
    M = 40
    Xq = np.ascontiguousarray(rng.random((M, 2)))
    mean = np.ascontiguousarray(rng.standard_normal(M))
    mgrad = np.ascontiguousarray(rng.standard_normal((M, 2)))
    s = 1.0 + 0.01
    for acq_id, ap in ((0, np.array([0.6, 0.0])), (1, np.array([0.2, 0.05]))):
        v, g = np.empty(M), np.empty((M, 2))
        assert lib.lb_acq_grad(h.h, acq_id, _p(ap), M, _p(Xq), _p(mean), 0.0, _p(mgrad), _p(v), _p(g)) == 0
        if acq_id == 0:
            rv, rg = AG.ucb(mean, np.full(M, s), mgrad, np.zeros((M, 2)), 0.6)
        else:
            rv, rg = AG.ei(mean, np.full(M, s), mgrad, np.zeros((M, 2)), 0.2, 0.05)
        assert np.allclose(v, rv, rtol=0, atol=1e-14) and np.allclose(g, rg, rtol=0, atol=1e-14)


def test_cpp_dropin():
    """tests/cpp/acq_grad_dropin_test.cpp: limbo_b200::acqui::UCB / EI gradients against central differences and the batched
    answer, the reference's opt::GradientAscent / opt::Adam over them, and limbo_b200::opt::BatchedGradient"""
    run_dropin("acq_grad_dropin_test", "ACQ GRAD DROPIN OK")
