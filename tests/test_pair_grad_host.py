"""The partials of oracle/pair_grad.py (ECI and two-objective EHVI with respect to each model's mu and sigma^2 / s) against central
differences of the restatements pinned to the reference (oracle.eci.eci_one, oracle.ehvi.ehvi2d), their chain through
oracle/acq_grad.query_grad against central differences in the candidate, and, where the reference's own ECI and ehvi2d are built
(oracle/_ref/libref_eci.so, libref_ehvi.so), the same checks against the reference's values.  CPU only."""
import math

import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky
from scipy.spatial.distance import cdist

from oracle import acq_grad as AG
from oracle import eci as OE
from oracle import ehvi as OH
from oracle import pair_grad as PG
from oracle import ref_eci, ref_ehvi

RTOL = 1e-6


def _fd(f, x, h):
    return (f(x + h) - f(x - h)) / (2 * h)


def _close(an, fd, scale):
    return abs(an - fd) <= RTOL * max(abs(an), abs(fd), scale)


def _eci_points(rng, n):
    """(mu0, s2, mu_c0, s2_c, f_max, jitter) with |Z| and |Z_c| below 3 and sigma well above the cut-offs"""
    return [(rng.uniform(-1, 1), rng.uniform(0.05, 1.0), rng.uniform(0.2, 1.8), rng.uniform(0.05, 1.0), rng.uniform(-0.5, 0.5),
             rng.choice([0.0, 0.01])) for _ in range(n)]


@pytest.mark.parametrize("con", ["model", "none", "empty"])
def test_eci_partials_match_central_differences(con):
    rng = np.random.default_rng(1)
    for mu0, s2, mc, sc, f_max, jit in _eci_points(rng, 40):
        con_empty = con == "empty"
        args = [mu0, s2, mc, sc]
        val, P = PG.eci_grad([mu0], [s2], None if con == "none" else [mc], None if con == "none" else [sc], f_max, jit,
                             con_empty=con_empty)

        def f(i, v):
            a = list(args)
            a[i] = v
            return OE.eci_one(a[0], a[1], a[2], a[3], f_max, jit, False, con_empty or con == "none")
        assert val[0] == f(0, mu0)
        for i in range(4):
            fd = _fd(lambda v: f(i, v), args[i], 1e-6 * max(1.0, abs(args[i])))
            assert _close(P[0, i], fd, 1e-3 * abs(val[0])), (con, i, P[0, i], fd)
        if con != "model":
            assert P[0, 2] == 0.0 and P[0, 3] == 0.0


def test_eci_cut_offs_give_zero_partials():
    _, P = PG.eci_grad([0.3], [1e-21], [1.0], [0.2], 0.0)
    assert np.all(P == 0.0)
    _, P = PG.eci_grad([0.3], [0.5], [1.0], [1e-21], 0.0)
    assert P[0, 0] > 0 and P[0, 2] == 0.0 and P[0, 3] == 0.0
    _, P = PG.eci_grad([0.3], [0.5], [1.0], [0.5], 0.0, obj_empty=True)
    assert np.all(P == 0.0)


def _front(rng, k):
    """k mutually non-dominated points (maximisation) in [0.1, 0.9]^2"""
    x = np.sort(rng.uniform(0.1, 0.9, k))
    y = np.sort(rng.uniform(0.1, 0.9, k))[::-1]
    return np.stack([x, y], axis=1)[rng.permutation(k)]


@pytest.mark.parametrize("k", [0, 1, 2, 5, 12])
def test_ehvi_partials_match_central_differences(k):
    rng = np.random.default_rng(10 + k)
    F = _front(rng, k)
    r = (-0.2, -0.1)
    checked = 0
    for _ in range(25):
        q = np.array([rng.uniform(-0.3, 1.2), rng.uniform(0.05, 0.6), rng.uniform(-0.3, 1.2), rng.uniform(0.05, 0.6)])
        val, P, mag, amb = PG.ehvi2d_grad(F, r, [q[0]], [q[1]], [q[2]], [q[3]])
        if np.any(amb > 0):  # a cell sign change at this point: no derivative to compare with
            continue
        assert abs(val[0] - OH.ehvi2d(F, r, (q[0], q[2]), (q[1], q[3]))) <= 1e-12 * max(1.0, abs(val[0]))

        def f(i, v):
            a = q.copy()
            a[i] = v
            return OH.ehvi2d(F, r, (a[0], a[2]), (a[1], a[3]))
        for i, col in enumerate((0, 1, 2, 3)):
            fd = _fd(lambda v: f(col, v), q[col], 1e-6)
            assert _close(P[0, i], fd, 1e-3 * (mag[0, i] + abs(val[0]) + 1.0)), (k, i, P[0, i], fd)
            assert mag[0, i] >= abs(P[0, i])
        checked += 1
    assert checked >= 15


def test_ehvi_value_is_the_table_form_and_dead_models_add_nothing():
    rng = np.random.default_rng(3)
    F = _front(rng, 9)
    m0, s0, m1, s1 = rng.uniform(0, 1, 30), rng.uniform(0.05, 0.5, 30), rng.uniform(0, 1, 30), rng.uniform(0.05, 0.5, 30)
    val, P, _, _ = PG.ehvi2d_grad(F, (0, 0), m0, s0, m1, s1)
    ref, _ = OH.ehvi2d_tables(F, (0, 0), m0, s0, m1, s1)
    assert np.allclose(val, ref, rtol=1e-12, atol=0)
    s0[:5] = 0.0
    _, P, _, _ = PG.ehvi2d_grad(F, (0, 0), m0, s0, m1, s1)
    assert np.all(P[:5, :2] == 0.0) and np.all(np.isfinite(P))


def _gp(kid, N, D, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    Y = (np.sin(3 * X[:, :1]) + X[:, -1:] ** 2 + shift)
    hp = np.concatenate([np.log(rng.uniform(0.3, 0.8, D)), [0.0]]) if kid == AG.K_SE_ARD else np.array([math.log(0.4), 0.0])
    J, sf2, l = AG.staging(kid, hp, D)
    K, _ = AG.kernel_and_coef(kid, cdist(X @ J, X @ J, "sqeuclidean"), sf2, l)
    K[np.diag_indices_from(K)] += 0.01 + 1e-8
    L = cholesky(K, lower=True)
    alpha = cho_solve((L, True), Y)
    return lambda Xq: AG.query_grad(kid, hp, 0.01, X, L, alpha, Xq)


def test_chains_match_central_differences_in_the_candidate():
    obj, con = _gp(AG.K_SE_ARD, 40, 2, 0), _gp(AG.K_MATERN52, 35, 2, 1, shift=0.8)
    rng = np.random.default_rng(5)
    Xq = rng.uniform(0.1, 0.9, (12, 2))
    F = _front(rng, 6)

    def eci_at(x):
        mo, so, dmo, dso, _ = obj(x)
        mc, sc, dmc, dsc, _ = con(x)
        val, P = PG.eci_grad(mo[:, 0], so, mc[:, 0], sc, 0.2, 0.0)
        return val, PG.chain(P, [dmo, dso, dmc, dsc])

    def ehvi_at(x):
        mo, so, dmo, dso, _ = obj(x)
        mc, sc, dmc, dsc, _ = con(x)
        val, P, _, amb = PG.ehvi2d_grad(F, (-0.5, -0.5), mo[:, 0], so, mc[:, 0], sc)
        return val, PG.chain(P, [dmo, dso, dmc, dsc]), amb
    for fun in (eci_at, ehvi_at):
        out = fun(Xq)
        val, g = out[0], out[1]
        ok = np.ones(len(Xq), bool) if fun is eci_at else ~np.any(out[2] > 0, axis=1)
        for d in range(2):
            e = np.zeros(2)
            e[d] = 1e-6
            fd = (fun(Xq + e)[0] - fun(Xq - e)[0]) / 2e-6
            scale = np.abs(g).max(axis=1) + 1e-8
            assert np.all((np.abs(g[:, d] - fd) <= RTOL * 10 * scale)[ok]), (fun.__name__, np.abs(g[:, d] - fd).max())


@pytest.mark.skipif(not ref_ehvi.available(), reason="the reference's ehvi2d is not built and its sources are not present")
def test_ehvi_partials_against_the_reference():
    rng = np.random.default_rng(7)
    F = _front(rng, 7)
    r = (-0.2, -0.1)
    for _ in range(20):
        q = np.array([rng.uniform(-0.3, 1.2), rng.uniform(0.05, 0.6), rng.uniform(-0.3, 1.2), rng.uniform(0.05, 0.6)])
        val, P, mag, amb = PG.ehvi2d_grad(F, r, [q[0]], [q[1]], [q[2]], [q[3]])
        if np.any(amb > 0):
            continue
        for i in range(4):
            h = np.zeros(4)
            h[i] = 1e-6
            vp, vm = (ref_ehvi.ehvi2d(F, r, [[a[0], a[2]]], [[a[1], a[3]]])[0] for a in (q + h, q - h))
            assert _close(P[0, i], (vp - vm) / 2e-6, 1e-3 * (mag[0, i] + abs(val[0]) + 1.0)), (i, P[0, i], (vp - vm) / 2e-6)


@pytest.mark.skipif(not ref_eci.available(), reason="the reference's ECI is not built and its sources are not present")
def test_eci_partials_against_the_reference():
    """the reference's ECI over its own GPs: d ECI / dx by central differences against the partials at its mu / sigma^2, chained
    with central differences of its own mu / sigma^2"""
    rng = np.random.default_rng(8)
    X = rng.random((30, 2))
    y = np.sin(3 * X[:, 0]) + X[:, 1]
    Yc = np.stack([1.0 + np.cos(2 * X[:, 0]), np.ones(30)], axis=1)
    Xq = rng.uniform(0.1, 0.9, (6, 2))
    base = ref_eci.eci(3, X, y, Yc, Xq)
    val, P = PG.eci_grad(base["mu"], base["sigma2"], base["mu_c"][:, 0], base["sigma2_c"], base["f_max"], 0.0)
    assert np.allclose(val, base["eci"], rtol=1e-12, atol=1e-15)
    h = 1e-6
    for d in range(2):
        e = np.zeros(2)
        e[d] = h
        p, m = ref_eci.eci(3, X, y, Yc, Xq + e), ref_eci.eci(3, X, y, Yc, Xq - e)
        fd = {k: (p[k] - m[k]) / (2 * h) for k in ("eci", "mu", "sigma2", "sigma2_c")}
        fd_mc = (p["mu_c"][:, 0] - m["mu_c"][:, 0]) / (2 * h)
        chained = P[:, 0] * fd["mu"] + P[:, 1] * fd["sigma2"] + P[:, 2] * fd_mc + P[:, 3] * fd["sigma2_c"]
        assert np.all(np.abs(chained - fd["eci"]) <= 1e-5 * (np.abs(fd["eci"]) + 1e-3 * np.abs(val) + 1e-9)), np.abs(chained - fd["eci"])
