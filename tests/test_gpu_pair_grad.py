"""Candidate gradients of the two-model acquisitions on the device (lb_eci_grad / lb_ehvi_grad): against the chain of
oracle/pair_grad.py's partials with oracle/acq_grad.py's grad mu / grad sigma^2, against lb_eci_argmax / lb_ehvi_argmax bit for bit
on the panel path, against central differences of the device's own argmax values, the edge cases, chunking at different widths on
the two handles, determinism, concurrent calls, plumbing (leases, errors), and bayes_opt.BatchedGradientSearch over ECI and EHVI."""
import ctypes as C
import gc
import math
import threading

import numpy as np
import pytest
from scipy.linalg import cho_solve, cholesky
from scipy.optimize import minimize
from scipy.spatial.distance import cdist

from dropin import run_dropin
from oracle import acq_grad as AG
from oracle import ehvi as OH
from oracle import pair_grad as PG

pytestmark = pytest.mark.gpu

LB_ERR_ARG, LB_ERR_UNSUPPORTED = -1, -5
TOL = 1e-9  # of the propagated per-candidate magnitude
EPS = np.finfo(np.float64).eps


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
        self.kid, self.hp, self.noise, self.X, self.Y = kid, np.asarray(hp, dtype=np.float64), noise, X, Y
        self.D, self.P = X.shape[1], Y.shape[1]
        self.L.check(self.lib.lb_set_data(self.h, X.shape[0], self.D, self.P, _p(X) if X.size else None, _p(Y) if Y.size else None), "set_data")
        hp = np.ascontiguousarray(hp, dtype=np.float64)
        self.L.check(self.lib.lb_set_kernel(self.h, kid, _p(hp), hp.size, noise), "set_kernel")
        if X.shape[0]:
            self.L.check(self.lib.lb_fit(self.h), "fit")

    def __del__(self):
        self.lib.lb_destroy(self.h)

    def reference(self, Xq):
        """oracle/acq_grad.py over K = k(X, X) + (noise + 1e-8) I, its SciPy factor and alpha: mu, s2, dmu, ds2, mag"""
        M = Xq.shape[0]
        if self.X.shape[0] == 0:
            _, sf2, _ = AG.staging(self.kid, self.hp, self.D)
            z = np.zeros((M, self.D))
            return np.zeros((M, 1)), np.full(M, sf2 + self.noise), z, z, z
        J, sf2, l = AG.staging(self.kid, self.hp, self.D)
        U = self.X @ J
        K, _ = AG.kernel_and_coef(self.kid, cdist(U, U, "sqeuclidean"), sf2, l)
        K[np.diag_indices_from(K)] += self.noise + 1e-8
        L = cholesky(K, lower=True)
        return AG.query_grad(self.kid, self.hp, self.noise, self.X, L, cho_solve((L, True), self.Y), Xq)


def eci_grad(o, c, Xq, f_max=0.2, jitter=0.0, means=None):
    Xq = np.ascontiguousarray(Xq, dtype=np.float64)
    M = Xq.shape[0]
    ep = np.array([f_max, jitter])
    m = means or {}
    v, g = np.empty(M), np.empty((M, o.D))
    rc = o.lib.lb_eci_grad(o.h, c.h if c else None, _p(ep), M, _p(Xq), _p(m.get("om")), m.get("oc", 0.0), _p(m.get("og")),
                           _p(m.get("cm")), m.get("cc", 0.0), _p(m.get("cg")), _p(v), _p(g))
    o.L.check(rc, "lb_eci_grad")
    return v, g


def eci_values(o, c, Xq, f_max=0.2, jitter=0.0):
    Xq = np.ascontiguousarray(Xq, dtype=np.float64)
    M = Xq.shape[0]
    ep = np.array([f_max, jitter])
    v, best, idx = np.empty(M), C.c_double(), C.c_int64()
    o.L.check(o.lib.lb_eci_argmax(o.h, c.h if c else None, _p(ep), M, _p(Xq), None, 0.0, None, 0.0, _p(v), C.addressof(best),
                                  C.addressof(idx)), "lb_eci_argmax")
    return v


def ehvi_grad(a, b, F, r, Xq, means=None):
    Xq = np.ascontiguousarray(Xq, dtype=np.float64)
    F = np.ascontiguousarray(np.asarray(F, dtype=np.float64).reshape(-1, 2))
    M = Xq.shape[0]
    rr = np.ascontiguousarray(r, dtype=np.float64)
    m = means or {}
    v, g = np.empty(M), np.empty((M, a.D))
    a.L.check(a.lib.lb_ehvi_grad(a.h, b.h, _p(rr), F.shape[0], _p(F) if F.size else None, M, _p(Xq), _p(m.get("om")), m.get("oc", 0.0),
                                 _p(m.get("og")), _p(m.get("cm")), m.get("cc", 0.0), _p(m.get("cg")), _p(v), _p(g)), "lb_ehvi_grad")
    return v, g


def ehvi_values(a, b, F, r, Xq):
    Xq = np.ascontiguousarray(Xq, dtype=np.float64)
    F = np.ascontiguousarray(np.asarray(F, dtype=np.float64).reshape(-1, 2))
    M = Xq.shape[0]
    rr = np.ascontiguousarray(r, dtype=np.float64)
    v, best, idx = np.empty(M), C.c_double(), C.c_int64()
    a.L.check(a.lib.lb_ehvi_argmax(a.h, b.h, _p(rr), F.shape[0], _p(F) if F.size else None, M, _p(Xq), None, 0.0, None, 0.0, _p(v),
                                   C.addressof(best), C.addressof(idx)), "lb_ehvi_argmax")
    return v


def _problem(kid, klam, N, D=3, P=1, seed=0, log_sf=0.0, noise=0.01, shift=0.0):
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    Y = np.stack([np.sin(3 * X[:, 0]) + X[:, -1] ** 2, np.cos(2 * X[:, 1])], axis=1)[:, :P]
    Y = Y - Y.mean(axis=0) + shift
    hp = np.concatenate([np.log(rng.uniform(0.3, 0.8, D)), 0.6 * rng.standard_normal(D * klam), [log_sf]]) if kid == AG.K_SE_ARD \
        else np.array([math.log(0.4), log_sf])
    return _Handle(kid, X, Y, hp, noise)


# (objective kernel, Lambda columns, P) and (constraint / second-objective kernel, Lambda columns): all four kernels, SE-ARD with
# Lambda, a different kernel on each handle, P > 1
PAIRS = [((AG.K_SE_ARD, 2, 2), (AG.K_MATERN32, 0)), ((AG.K_MATERN52, 0, 1), (AG.K_EXP, 0)), ((AG.K_EXP, 0, 2), (AG.K_SE_ARD, 0)),
         ((AG.K_MATERN32, 0, 1), (AG.K_MATERN52, 0))]


def _pair(i, N0=600, N1=450):
    (k0, l0, p0), (k1, l1) = PAIRS[i]
    return _problem(k0, l0, N0, P=p0, seed=i), _problem(k1, l1, N1, seed=10 + i, shift=0.9)


def _eci_tol(P, mo, mc):
    return TOL * ((np.abs(P[:, :1]) + np.abs(P[:, 1:2])) * mo + (np.abs(P[:, 2:3]) + np.abs(P[:, 3:4])) * mc) + 1e-15


@pytest.mark.parametrize("i", range(len(PAIRS)))
def test_eci_against_the_oracle_chain(i):
    o, c = _pair(i)
    Xq = np.random.default_rng(20 + i).random((300, 3))
    for con in (c, None):
        v, g = eci_grad(o, con, Xq, f_max=0.1, jitter=0.01)
        mo, so, dmo, dso, mago = o.reference(Xq)
        if con is None:
            rv, P = PG.eci_grad(mo[:, 0], so, None, None, 0.1, 0.01)
            rg, magc = PG.chain(P, [dmo, dso, 0 * dmo, 0 * dso]), 0 * mago
        else:
            mc, sc, dmc, dsc, magc = c.reference(Xq)
            rv, P = PG.eci_grad(mo[:, 0], so, mc[:, 0], sc, 0.1, 0.01)
            rg = PG.chain(P, [dmo, dso, dmc, dsc])
        assert np.allclose(v, rv, rtol=0, atol=1e-10)
        err = np.abs(g - rg)
        tol = _eci_tol(P, mago, magc)
        assert np.all(err <= tol), (err / tol).max()
        print(f"ECIGRAD pair={i} con={con is not None} max|err|/tol={(err / tol).max():.3e}")


def _ehvi_tol(P, pmag, amb, grads, mags):
    tol = 1e-15
    for q, (gx, mg) in enumerate(zip(grads, mags)):
        tol = tol + TOL * np.abs(P[:, q:q + 1]) * mg + (64 * EPS * pmag[:, q:q + 1] + amb[:, q:q + 1]) * np.abs(gx)
    return tol


def _front(rng, k, lo=-0.8, hi=0.8):
    x = np.sort(rng.uniform(lo, hi, k))
    y = np.sort(rng.uniform(lo, hi, k))[::-1]
    return np.stack([x, y], axis=1)[rng.permutation(k)]


@pytest.mark.parametrize("k", [0, 1, 40, 4096])
@pytest.mark.parametrize("i", [0, 1])
def test_ehvi_against_the_oracle_chain(i, k):
    a, b = _pair(i)
    rng = np.random.default_rng(30 + k)
    Xq = rng.random((8 if k == 4096 else 300, 3))
    F = _front(rng, k)
    r = (-1.5, -1.2)
    v, g = ehvi_grad(a, b, F, r, Xq)
    m0, s0, d0, e0, g0 = a.reference(Xq)
    m1, s1, d1, e1, g1 = b.reference(Xq)
    rv, P, pmag, amb = PG.ehvi2d_grad(F, r, m0[:, 0], s0, m1[:, 0], s1)
    vt, vscale = OH.ehvi2d_tables(F, r, m0[:, 0], s0, m1[:, 0], s1)
    assert np.all(np.abs(v - rv) <= OH.tolerance(rv, vscale) + 1e-9 * np.abs(rv) + 1e-12)
    rg = PG.chain(P, [d0, e0, d1, e1])
    tol = _ehvi_tol(P, pmag, amb, [d0, e0, d1, e1], [g0, g0, g1, g1])
    err = np.abs(g - rg)
    assert np.all(err <= tol), (err / tol).max()
    print(f"EHVIGRAD pair={i} k={k} max|err|/tol={(err / tol).max():.3e}")


def test_input_dependent_means_on_both_models():
    """per-candidate mean arrays and mean gradients on both models (distinct on each, so that a swapped model or a wrong offset
    shows), against the oracle chain with each mean's gradient added to its model's grad mu"""
    o, c = _pair(0)
    rng = np.random.default_rng(25)
    Xq = rng.random((300, 3))
    om, cm = 0.3 * np.sin(4 * Xq[:, 0]), 0.5 + 0.2 * Xq[:, 1] ** 2
    og = np.stack([1.2 * np.cos(4 * Xq[:, 0]), 0 * Xq[:, 0], 0 * Xq[:, 0]], axis=1)
    cg = np.stack([0 * Xq[:, 1], 0.4 * Xq[:, 1], 0.1 + 0 * Xq[:, 2]], axis=1)
    means = {"om": np.ascontiguousarray(om), "og": np.ascontiguousarray(og), "cm": np.ascontiguousarray(cm),
             "cg": np.ascontiguousarray(cg), "oc": 7.0, "cc": -7.0}  # the constants are ignored next to the arrays
    mo, so, dmo, dso, mago = o.reference(Xq)
    mc, sc, dmc, dsc, magc = c.reference(Xq)
    v, g = eci_grad(o, c, Xq, f_max=0.1, means=means)
    rv, P = PG.eci_grad(mo[:, 0] + om, so, mc[:, 0] + cm, sc, 0.1)
    rg = PG.chain(P, [dmo + og, dso, dmc + cg, dsc])
    assert np.allclose(v, rv, rtol=0, atol=1e-10)
    assert np.all(np.abs(g - rg) <= _eci_tol(P, mago + np.abs(og), magc + np.abs(cg)))
    F, r = _front(rng, 25), (-1.5, -1.2)
    v, g = ehvi_grad(o, c, F, r, Xq, means=means)
    rv, P, pmag, amb = PG.ehvi2d_grad(F, r, mo[:, 0] + om, so, mc[:, 0] + cm, sc)
    _, vscale = OH.ehvi2d_tables(F, r, mo[:, 0] + om, so, mc[:, 0] + cm, sc)
    assert np.all(np.abs(v - rv) <= OH.tolerance(rv, vscale) + 1e-9 * np.abs(rv) + 1e-12)
    grads = [dmo + og, dso, dmc + cg, dsc]
    tol = _ehvi_tol(P, pmag, amb, grads, [mago + np.abs(og), mago, magc + np.abs(cg), magc])
    assert np.all(np.abs(g - PG.chain(P, grads)) <= tol)
    # the constant-mean form: a constant array equals the constant
    const = {"oc": 0.25, "cc": -0.4}
    arr = {"om": np.full(300, 0.25), "cm": np.full(300, -0.4)}
    for call in (lambda m: eci_grad(o, c, Xq, means=m), lambda m: ehvi_grad(o, c, F, r, Xq, means=m)):
        a, b = call(const), call(arr)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("i", range(len(PAIRS)))
def test_values_equal_the_argmax_values(i):
    o, c = _pair(i)
    rng = np.random.default_rng(40 + i)
    Xq = rng.random((300, 3))
    for con in (c, None):
        assert np.array_equal(eci_grad(o, con, Xq)[0], eci_values(o, con, Xq))
    for k in (0, 1, 4096):
        F = _front(rng, k)
        assert np.array_equal(ehvi_grad(o, c, F, (-1.5, -1.2), Xq)[0], ehvi_values(o, c, F, (-1.5, -1.2), Xq))


def test_central_differences_of_the_device_values():
    L, lib = _lib()
    o, c = _pair(0)
    Xq = np.random.default_rng(50).random((8, 3))
    F = _front(np.random.default_rng(51), 12)
    lib.lb_debug_set_query_panel_min(1)  # the argmax values on the panel path at 8 candidates
    try:
        for grad, vals in ((lambda x: eci_grad(o, c, x), lambda x: eci_values(o, c, x)),
                           (lambda x: ehvi_grad(o, c, F, (-1.5, -1.2), x), lambda x: ehvi_values(o, c, F, (-1.5, -1.2), x))):
            v, g = grad(Xq)
            assert np.array_equal(v, vals(Xq))
            H = 1e-5
            for d in range(3):
                e = np.zeros(3)
                e[d] = H
                fd = (vals(Xq + e) - vals(Xq - e)) / (2 * H)
                scale = np.maximum(np.abs(g).max(axis=1), 1e-3)
                assert np.all(np.abs(g[:, d] - fd) <= 1e-6 * scale), np.abs(g[:, d] - fd).max()
    finally:
        lib.lb_debug_set_query_panel_min(0)


def test_eci_edge_cases():
    o, c = _pair(1)
    Xq = np.vstack([o.X[:3], np.random.default_rng(60).random((300, 3))])
    # a constraint without samples: Pf = 1, as with no constraint handle
    empty = _Handle(AG.K_EXP, np.zeros((0, 3)), np.zeros((0, 1)), [math.log(0.4), 0.0], 0.01)
    assert all(np.array_equal(x, y) for x, y in zip(eci_grad(o, empty, Xq), eci_grad(o, None, Xq)))
    # an objective without samples: 0 everywhere
    v, g = eci_grad(empty, c, Xq)
    assert np.all(v == 0.0) and np.all(g == 0.0)
    # sigma_f^2 = e^-40 with noise 0: the clamp is active everywhere, sigma = 0 < 1e-10 on either model
    tiny_o = _problem(AG.K_SE_ARD, 0, 200, log_sf=-20.0, noise=0.0)
    tiny_c = _problem(AG.K_MATERN52, 0, 150, seed=3, log_sf=-20.0, noise=0.0, shift=0.5)
    v, g = eci_grad(tiny_o, c, Xq)
    assert np.all(v == 0.0) and np.all(g == 0.0)
    v, g = eci_grad(o, tiny_c, Xq)
    v1, g1 = eci_grad(o, None, Xq)
    assert np.array_equal(v, v1) and np.array_equal(g, g1)
    # an active clamp with noise > 0 (sigma above the cut-off): grad sigma^2 = 0 leaves Pf grad EI's mean term
    clamp = _problem(AG.K_SE_ARD, 0, 200, log_sf=-20.0, noise=0.01)
    v, g = eci_grad(clamp, None, Xq)
    mo, so, dmo, dso, mago = clamp.reference(Xq)
    rv, P = PG.eci_grad(mo[:, 0], so, None, None, 0.2)
    assert np.all(dso == 0.0) and np.allclose(v, rv, rtol=0, atol=1e-12)
    assert np.all(np.abs(g - PG.chain(P, [dmo, dso, 0 * dmo, 0 * dso])) <= _eci_tol(P, mago, 0 * mago))


def test_ehvi_edge_cases():
    a, b = _pair(2)
    rng = np.random.default_rng(70)
    Xq = rng.random((300, 3))
    r = (-1.5, -1.2)
    # coincident front points: the same as the front without the copies
    F = _front(rng, 9)
    v, g = ehvi_grad(a, b, np.vstack([F, F[:3]]), r, Xq)
    assert np.array_equal(v, ehvi_values(a, b, np.vstack([F, F[:3]]), r, Xq))
    assert np.all(np.isfinite(g))
    # cells with sum <= 0: a front far above the candidates' means leaves many cells with a non-positive sum
    far = _front(rng, 30, 3.0, 6.0)
    m0, s0, d0, e0, g0 = a.reference(Xq)
    m1, s1, d1, e1, g1 = b.reference(Xq)
    v, g = ehvi_grad(a, b, far, r, Xq)
    rv, P, pmag, amb = PG.ehvi2d_grad(far, r, m0[:, 0], s0, m1[:, 0], s1)
    err = np.abs(g - PG.chain(P, [d0, e0, d1, e1]))
    assert np.all(err <= _ehvi_tol(P, pmag, amb, [d0, e0, d1, e1], [g0, g0, g1, g1]))
    # one model at its prior: zero grad mu / grad sigma^2 there, only the other model's gradient remains
    prior = _Handle(AG.K_MATERN52, np.zeros((0, 3)), np.zeros((0, 1)), [math.log(0.4), 0.0], 0.01)
    v, g = ehvi_grad(a, prior, F, r, Xq)
    assert np.array_equal(v, ehvi_values(a, prior, F, r, Xq))
    mp, sp, dp, ep, gp = prior.reference(Xq)
    rv, P, pmag, amb = PG.ehvi2d_grad(F, r, m0[:, 0], s0, mp[:, 0], sp)
    err = np.abs(g - PG.chain(P, [d0, e0, dp, ep]))
    assert np.all(err <= _ehvi_tol(P, pmag, amb, [d0, e0, dp, ep], [g0, g0, gp, gp]))


def test_chunks_at_different_widths_on_the_two_handles():
    """one handle at N = 16384 splits 50000 candidates at its 6 GiB chunk (49152); the other takes them in one chunk"""
    big = _problem(AG.K_MATERN52, 0, 16384, D=6, seed=80)
    small = _problem(AG.K_SE_ARD, 0, 3000, D=6, seed=81, shift=0.9)
    Xq = np.random.default_rng(82).random((50000, 6))
    v, g = eci_grad(big, small, Xq)
    assert np.array_equal(v, eci_values(big, small, Xq))
    F = _front(np.random.default_rng(83), 16)
    v2, g2 = ehvi_grad(small, big, F, (-1.5, -1.2), Xq)
    assert np.array_equal(v2, ehvi_values(small, big, F, (-1.5, -1.2), Xq))
    # the candidates on each side of the chunk boundary against single-handle gradients chained on the host
    sel = np.r_[49100:49200]
    mu_b, s_b, dmu_b, ds_b = (np.empty((50000, 1)), np.empty(50000), np.empty((50000, 6)), np.empty((50000, 6)))
    big.L.check(big.lib.lb_query_grad(big.h, 50000, _p(np.ascontiguousarray(Xq)), _p(mu_b), _p(s_b), _p(dmu_b), _p(ds_b)), "qg")
    mu_s, s_s, dmu_s, ds_s = (np.empty((50000, 1)), np.empty(50000), np.empty((50000, 6)), np.empty((50000, 6)))
    small.L.check(small.lib.lb_query_grad(small.h, 50000, _p(np.ascontiguousarray(Xq)), _p(mu_s), _p(s_s), _p(dmu_s), _p(ds_s)), "qg")
    rv, P = PG.eci_grad(mu_b[sel, 0], s_b[sel], mu_s[sel, 0], s_s[sel], 0.2)
    rg = PG.chain(P, [dmu_b[sel], ds_b[sel], dmu_s[sel], ds_s[sel]])
    assert np.allclose(v[sel], rv, rtol=1e-13, atol=1e-15)
    assert np.allclose(g[sel], rg, rtol=1e-12, atol=1e-12 * np.abs(rg).max())


def test_bits_do_not_depend_on_the_batch_or_the_call():
    o, c = _pair(3)
    rng = np.random.default_rng(90)
    Xq = rng.random((400, 3))
    F = _front(rng, 33)
    perm = rng.permutation(400)
    for call in (lambda x: eci_grad(o, c, x), lambda x: ehvi_grad(o, c, F, (-1.5, -1.2), x)):
        a, b = call(Xq), call(Xq)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
        p = call(Xq[perm])
        assert all(np.array_equal(x[perm], y) for x, y in zip(a, p))


def test_two_threads_with_the_roles_swapped():
    o, c = _pair(1, N0=1500, N1=1300)
    rng = np.random.default_rng(91)
    Xq = rng.random((512, 3))
    F = _front(rng, 20)
    calls = [lambda: eci_grad(o, c, Xq), lambda: eci_grad(c, o, Xq), lambda: ehvi_grad(o, c, F, (-1.5, -1.2), Xq),
             lambda: ehvi_grad(c, o, F, (-1.5, -1.2), Xq)]
    serial = [f() for f in calls]
    results, errors = {}, []

    def run(j):
        try:
            for it in range(6):
                results[(j, it)] = calls[(j + it) % 4]()
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)
    ts = [threading.Thread(target=run, args=(j,)) for j in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for (j, it), r in results.items():
        assert all(np.array_equal(x, y) for x, y in zip(r, serial[(j + it) % 4]))


def _round():
    from limbo_b200 import acqui, kernel, model
    rng = np.random.default_rng(92)
    X = rng.random((150, 2))
    gp = model.GP(2, 1, kernel=kernel.SquaredExpARD)
    gp.compute(X, np.sin(4 * X[:, :1]))
    con = model.GP(2, 1, kernel=kernel.Exp)
    con.compute(X, 1.0 + np.cos(3 * X[:, 1:]))
    Xq = rng.random((400, 2))
    acqui.ECI(gp, con).grad_batch(Xq)
    acqui.ECI(gp, None)(Xq[0], gradient=True)
    e = acqui.EHVI([gp, con], np.array([[0.5, 1.5], [0.9, 1.0]]), (-1.0, -1.0))
    e.grad_batch(Xq)
    e(Xq[1], gradient=True)
    del gp, con, e


def test_round_returns_every_lease():
    L, lib = _lib()
    _round()
    gc.collect()
    live = lib.lb_debug_pool_live()
    _round()
    gc.collect()
    assert lib.lb_debug_pool_live() == live


def test_errors():
    o, c = _pair(1, N0=100, N1=90)
    lib = o.lib
    Xq = np.random.default_rng(93).random((4, 3))
    v, g = np.empty(4), np.empty((4, 3))
    ep, r = np.array([0.1, 0.0]), np.array([-1.0, -1.0])
    F = np.array([[0.2, 0.5], [0.4, 0.1]])

    def eci(obj, con, M=4, X=Xq):
        return lib.lb_eci_grad(obj.h, con.h if con else None, _p(ep), M, _p(X), None, 0.0, None, None, 0.0, None, _p(v), _p(g))

    def ehvi(a, b, M=4, X=Xq, k=2, front=F, rr=r):
        return lib.lb_ehvi_grad(a.h, b.h, _p(rr), k, _p(front), M, _p(X), None, 0.0, None, None, 0.0, None, _p(v), _p(g))
    assert eci(o, o) == LB_ERR_ARG and ehvi(o, o) == LB_ERR_ARG
    assert eci(o, c, M=0) == LB_ERR_ARG and ehvi(o, c, M=0) == LB_ERR_ARG
    bad = Xq.copy()
    bad[1, 2] = np.inf
    assert eci(o, c, X=bad) == LB_ERR_ARG and ehvi(o, c, X=bad) == LB_ERR_ARG
    assert ehvi(o, c, front=np.array([[0.2, np.nan], [0.4, 0.1]])) == LB_ERR_ARG
    assert ehvi(o, c, rr=np.array([np.inf, 0.0])) == LB_ERR_ARG
    big = np.zeros((4097, 2))
    assert ehvi(o, c, k=4097, front=big) == LB_ERR_UNSUPPORTED
    d2 = _problem(AG.K_EXP, 0, 50, D=2, seed=94)
    assert eci(o, d2) == LB_ERR_ARG and ehvi(o, d2) == LB_ERR_ARG
    tf = _problem(AG.K_MATERN32, 0, 100, seed=95)
    tf32 = _Handle(AG.K_MATERN32, tf.X, tf.Y, tf.hp, 0.01, precision=1)
    assert eci(tf32, c) == LB_ERR_UNSUPPORTED and eci(o, tf32) == LB_ERR_UNSUPPORTED
    assert ehvi(tf32, c) == LB_ERR_UNSUPPORTED and ehvi(o, tf32) == LB_ERR_UNSUPPORTED


class _OptParams:
    class acqui_eci:
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


def _oracle_fit(O, gp, X, y):
    kid = gp.kernel_function().kernel_id
    hp = np.asarray(gp.kernel_function().params(), dtype=np.float64)
    og = O.OracleGP()
    og.set_data(X, y - y.mean())
    og.set_kernel(kid, hp, gp.kernel_function().noise())
    og.fit()
    Lo, ao = og.get(1), og.get(2)
    return lambda x: AG.query_grad(kid, hp, og.noise, X, Lo, ao, np.atleast_2d(x)), float(y.mean()), og


@pytest.mark.parametrize("acq_name", ["ECI", "EHVI"])
def test_gradient_search_reaches_the_lbfgsb_maximum(acq_name, oracle_mod):
    from limbo_b200 import acqui, bayes_opt, kernel, mean, model
    rng = np.random.default_rng(96)
    X = rng.random((60, 2))
    y0 = np.sin(5 * X[:, :1]) * np.cos(3 * X[:, 1:]) + 0.3 * X[:, :1]
    y1 = 1.0 + np.cos(4 * X[:, :1] + X[:, 1:]) if acq_name == "ECI" else np.cos(3 * X[:, :1]) - 0.5 * X[:, 1:]
    g0 = model.GP(2, 1, params=_OptParams, kernel=kernel.SquaredExpARD, mean=mean.Data)
    g1 = model.GP(2, 1, params=_OptParams, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    g0.compute(X, y0)
    g1.compute(X, y1)
    q0, c0, og0 = _oracle_fit(oracle_mod, g0, X, y0)
    q1, c1, _ = _oracle_fit(oracle_mod, g1, X, y1)
    if acq_name == "ECI":
        acq = acqui.ECI(g0, g1, 0, params=_OptParams)
        f_max = float(og0.query(X)[0][:, 0].max() + c0)
    else:
        from limbo_b200 import pareto
        pop = np.array([p[1] for p in pareto.pareto_set(list(zip(X, np.hstack([y0, y1]), [np.zeros(2)] * 60)), 1)])
        acq = acqui.EHVI([g0, g1], pop, (-1.5, -1.5))

    def neg(x):
        m0, s0, d0, e0, _ = q0(x)
        m1, s1, d1, e1, _ = q1(x)
        if acq_name == "ECI":
            v, P = PG.eci_grad(m0[:, 0] + c0, s0, m1[:, 0] + c1, s1, f_max, 0.0)
        else:
            v, P, _, _ = PG.ehvi2d_grad(pop, (-1.5, -1.5), m0[:, 0] + c0, s0, m1[:, 0] + c1, s1)
        return -float(v[0]), -PG.chain(P, [d0, e0, d1, e1])[0]
    starts = np.vstack([rng.random((40, 2)), np.stack(np.meshgrid(np.linspace(0.05, 0.95, 6), np.linspace(0.05, 0.95, 6)), -1).reshape(-1, 2)])
    best = max(-minimize(neg, s, jac=True, method="L-BFGS-B", bounds=[(0, 1), (0, 1)], options={"ftol": 1e-15, "gtol": 1e-12}).fun
               for s in starts)
    xg = bayes_opt.BatchedGradientSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    xr = bayes_opt.BatchedRandomSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    vg, vr = acq.grad_batch(np.vstack([xg, xr]))[0]
    print(f"GRADSEARCH {acq_name} gradient={vg:.12g} random={vr:.12g} lbfgsb={best:.12g}")
    assert vg >= best - 1e-6, (vg, best)
    assert vg >= vr


def test_cboptimizer_and_ehvi_run_with_the_gradient_search():
    from limbo_b200 import bayes_opt, kernel, mean, model

    class P(_OptParams):
        class kernel:
            noise = 1e-6

        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 10

        class opt_batchedgradient:
            candidates = 2000
            starts = 16
            iterations = 30
            alpha = 0.01

    def f(x):
        return np.array([-float(((x - np.array([0.25, 0.75])) ** 2).sum()), 1.0 if x[0] + x[1] >= 1.2 else 0.0])
    gp = model.GP(2, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    con = model.GP(2, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Constant)
    bo = bayes_opt.CBOptimizer(gp, con, params=P, acqui_opt=bayes_opt.BatchedGradientSearch(P, np.random.default_rng(1)),
                               rng=np.random.default_rng(1))
    bo.optimize(f, 2, dim_out=1, nb_constraints=1)
    assert len(bo.samples()) == 20 and all(np.all((s >= 0) & (s <= 1)) for s in bo.samples())
    mo = bayes_opt.Ehvi(params=P, acqui_opt=bayes_opt.BatchedGradientSearch(P, np.random.default_rng(2)), rng=np.random.default_rng(2))
    mo.optimize(lambda x: OH.mop2(x)[0], 2)
    assert len(mo.samples()) == 20 and all(np.all(np.isfinite(s)) and np.all((s >= 0) & (s <= 1)) for s in mo.samples())


def test_cpp_dropin():
    """tests/cpp/pair_grad_dropin_test.cpp: limbo_b200::acqui::ECI gradients against central differences and the batched answer,
    the reference's opt::Adam over them, and limbo_b200::opt::BatchedGradient in the inner loops of CBOptimizer and Ehvi over
    limbo_b200::acqui::ECI and the acqui::Ehvi specialisation"""
    run_dropin("pair_grad_dropin_test", "PAIR GRAD DROPIN OK")
