"""Candidate gradients of the pseudo-input sparse GP on the device (lb_spgp_query_grad / lb_spgp_acq_grad, limbo_b200/csrc/spgp.cu)
against the NumPy gradients of oracle/spgp_grad.py, bounded by the per-entry magnitude sqrt(b_d) sum_m k_m |x~_d - x~b_md|
(|b1_m| + 2 |u_m|): up to N = 16384, M = 1638, D = 6, across two candidate chunks, and on the reference fixtures of
tests/golden/spgp.  Also: bit-identity with lb_spgp_query / lb_spgp_acq_argmax, repeat calls and two threads, the optimized flag,
the error codes, an input-dependent mean, model.SPGP under acqui.UCB / EI and bayes_opt.BatchedGradientSearch, and the C++
drop-in test."""
import ctypes as C
import glob
import math
import os
import threading

import numpy as np
import pytest
from scipy.optimize import minimize

from dropin import run_dropin
from oracle import acq_grad as AG
from oracle import spgp as O
from oracle import spgp_grad as SG

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "spgp", "*.npz")))
LB_ERR_ARG, LB_ERR_STATE = -1, -3
JITTER = 1e-6
BOUND = 1e-9
QCHUNK = 8192


def _p(a):
    return None if a is None else a.ctypes.data


class Raw:
    """lb_spgp handle over the raw ABI."""

    def __init__(self):
        from limbo_b200 import _lib
        self.lib = _lib.load()
        self.h = C.c_void_p()
        assert self.lib.lb_spgp_create(C.byref(self.h), 0) == 0

    def __del__(self):
        self.lib.lb_spgp_destroy(self.h)

    def fit(self, X, y, M, w, jitter=JITTER):
        X = np.ascontiguousarray(X, dtype=np.float64)
        y = np.ascontiguousarray(y, dtype=np.float64)
        w = np.ascontiguousarray(w, dtype=np.float64)
        assert self.lib.lb_spgp_set_data(self.h, X.shape[0], X.shape[1], _p(X), _p(y)) == 0
        assert self.lib.lb_spgp_compute(self.h, M, w.size, _p(w), jitter) == 0

    def query(self, Xq, optimized=1):
        mu, s2 = np.full(len(Xq), np.nan), np.full(len(Xq), np.nan)
        assert self.lib.lb_spgp_query(self.h, len(Xq), _p(Xq), optimized, _p(mu), _p(s2)) == 0
        return mu, s2

    def argmax_values(self, acq_id, ap, Xq, optimized=1, mean=None, mconst=0.0):
        vals = np.full(len(Xq), np.nan)
        best, idx = C.c_double(), C.c_int64(-1)
        assert self.lib.lb_spgp_acq_argmax(self.h, acq_id, _p(ap), len(Xq), _p(Xq), optimized, _p(mean), mconst, _p(vals),
                                           C.addressof(best), C.addressof(idx)) == 0
        return vals

    def query_grad(self, Xq, optimized=1):
        M, D = Xq.shape
        mu, s2, dmu, ds2 = np.full(M, np.nan), np.full(M, np.nan), np.full((M, D), np.nan), np.full((M, D), np.nan)
        rc = self.lib.lb_spgp_query_grad(self.h, M, _p(Xq), optimized, _p(mu), _p(s2), _p(dmu), _p(ds2))
        assert rc == 0, rc
        return mu, s2, dmu, ds2

    def acq_grad(self, acq_id, ap, Xq, optimized=1, mean=None, mconst=0.0, mgrad=None):
        M, D = Xq.shape
        v, g = np.full(M, np.nan), np.full((M, D), np.nan)
        rc = self.lib.lb_spgp_acq_grad(self.h, acq_id, _p(ap), M, _p(Xq), optimized, _p(mean), mconst, _p(mgrad), _p(v), _p(g))
        assert rc == 0, rc
        return v, g


def _case(seed, N, D, M=None, hartmann=False):
    from limbo_b200 import synth
    rng = np.random.default_rng(seed)
    if hartmann:
        X = synth.points(seed, N, D)
        y = synth.targets(X)
    else:
        X = rng.random((N, D))
        y = np.sin(3.0 * X).sum(axis=1) + 0.05 * rng.normal(size=N)
    y = y - y.mean()
    M = O.n_pseudo(N) if M is None else M
    w = O.init_w(X, y, M, rng.permutation(N)) + rng.normal(0.0, 0.05, (M + 1) * D + 2)
    return X, y, M, w


def _check_against_oracle(s, st, Xq, rows, label):
    """device gradients on all of Xq, the oracle on `rows`; returns the largest error / bound over every quantity"""
    mu, s2, dmu, ds2 = s.query_grad(Xq)
    mq, sq = s.query(Xq)
    assert np.array_equal(mu, mq) and np.array_equal(s2, sq)
    f_max = float(mu.max()) - 0.05
    aps = {0: np.array([0.5, 0.0]), 1: np.array([f_max, 0.01])}
    acq = {}
    for acq_id, ap in aps.items():
        v, g = s.acq_grad(acq_id, ap, Xq)
        assert np.array_equal(v, s.argmax_values(acq_id, ap, Xq)), acq_id
        acq[acq_id] = (v, g)
    worst = 0.0
    for r0 in range(0, len(rows), 512):
        r = rows[r0:r0 + 512]
        mo, so, dmo, dso, mag = SG.query_grad(st, Xq[r])
        bound = BOUND * mag + 1e-300
        for name, dev, ref, b in (("dmu", dmu[r], dmo, bound), ("ds2", ds2[r], dso, bound)):
            e = float((np.abs(dev - ref) / b).max())
            assert e <= 1.0, (label, name, e)
            worst = max(worst, e)
        sq_ = np.sqrt(so)
        ucb_v, ucb_g = AG.ucb(mo, so, dmo, dso, 0.5)
        e = float((np.abs(acq[0][1][r] - ucb_g) / (bound * (1.0 + 0.5 / (2.0 * sq_))[:, None])).max())
        assert e <= 1.0, (label, "ucb", e)
        worst = max(worst, e)
        ei_v, ei_g = AG.ei(mo, so, dmo, dso, f_max, 0.01)
        e = float((np.abs(acq[1][1][r] - ei_g) / (bound * (1.0 + 1.0 / (2.0 * sq_))[:, None])).max())
        assert e <= 1.0, (label, "ei", e)
        worst = max(worst, e)
    print(f"{label}: largest error / bound {worst:.3e}")
    return worst


@pytest.mark.parametrize("seed,N,D,M,Mq,hartmann", [
    (7, 16384, 6, 1638, QCHUNK + 37, True),  # the headline shape, two chunks, the second a partial tile
    (2, 2000, 3, 201, 700, False),           # M not a multiple of 128
    (3, 300, 2, 1, 300, False),              # one pseudo-input
    (4, 3000, 5, 300, QCHUNK + 37, False),
])
def test_gradients_against_the_oracle(seed, N, D, M, Mq, hartmann):
    X, y, M, w = _case(seed, N, D, M, hartmann)
    s = Raw()
    s.fit(X, y, M, w)
    st = O.State(w, X, y, M, JITTER)
    rng = np.random.default_rng(seed + 100)
    Xq = np.ascontiguousarray(np.vstack([rng.random((Mq - 20, D)), rng.random((20, D)) * 3.0 - 1.0]))
    rows = np.unique(np.concatenate([np.arange(min(Mq, 600)), np.arange(max(0, QCHUNK - 64), min(Mq, QCHUNK + 64)),
                                     np.arange(max(0, Mq - 80), Mq)]))
    _check_against_oracle(s, st, Xq, rows, f"N={N} M={M} D={D} Mq={Mq}")


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_gradients_on_the_reference_fixtures(path):
    g = np.load(path)
    X, y, M, w, jit, Xq = g["X"], g["y"], int(g["M"]), g["w"], float(g["jitter"]), np.ascontiguousarray(g["Xq"])
    s = Raw()
    s.fit(X, y - y.mean(), M, w, jitter=jit)
    st = O.State(w, X, y - y.mean(), M, jit)
    _check_against_oracle(s, st, Xq, np.arange(len(Xq)), os.path.basename(path))


def _small():
    X, y, M, w = _case(5, 400, 3, 40)
    s = Raw()
    s.fit(X, y, M, w)
    Xq = np.ascontiguousarray(np.random.default_rng(9).random((300, 3)))
    return s, X, y, M, w, Xq


def test_repeat_calls_and_two_threads_are_bit_identical():
    s, _, _, _, _, Xq = _small()
    a = s.query_grad(Xq)
    b = s.query_grad(Xq)
    assert all(np.array_equal(p, q) for p, q in zip(a, b))
    ap = np.array([0.2, 0.01])
    ga = s.acq_grad(1, ap, Xq)
    assert all(np.array_equal(p, q) for p, q in zip(ga, s.acq_grad(1, ap, Xq)))
    # one candidate's result does not depend on the rest of the batch
    part = s.query_grad(np.ascontiguousarray(Xq[100:130]))
    assert all(np.array_equal(p[100:130], q) for p, q in zip(a, part))
    out = {}

    def work(k):
        out[k] = [s.query_grad(Xq) for _ in range(3)] + [s.acq_grad(1, ap, Xq)]
    ts = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for k in range(2):
        for r in out[k][:3]:
            assert all(np.array_equal(p, q) for p, q in zip(a, r))
        assert all(np.array_equal(p, q) for p, q in zip(ga, out[k][3]))


def test_optimized_flag_moves_sigma2_only():
    s, _, _, M, w, Xq = _small()
    a = s.query_grad(Xq, optimized=0)
    b = s.query_grad(Xq, optimized=1)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
    assert np.array_equal(b[1], s.query(Xq, optimized=1)[1]) and np.array_equal(a[1], s.query(Xq, optimized=0)[1])


def test_error_codes():
    s, X, y, M, w, Xq = _small()
    lib = s.lib
    D = 3
    ap = np.array([0.5, 0.0])
    o = np.empty((4, D))
    v = np.empty(4)
    assert lib.lb_spgp_query_grad(None, 4, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_ARG
    assert lib.lb_spgp_query_grad(s.h, 0, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_ARG
    assert lib.lb_spgp_query_grad(s.h, -3, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_ARG
    assert lib.lb_spgp_query_grad(s.h, 4, None, 1, None, None, _p(o), None) == LB_ERR_ARG
    bad = np.ascontiguousarray(Xq[:4].copy())
    bad[2, 1] = np.nan
    assert lib.lb_spgp_query_grad(s.h, 4, _p(bad), 1, None, None, _p(o), None) == LB_ERR_ARG
    bad[2, 1] = np.inf
    assert lib.lb_spgp_acq_grad(s.h, 0, _p(ap), 4, _p(bad), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    assert lib.lb_spgp_acq_grad(None, 0, _p(ap), 4, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    assert lib.lb_spgp_acq_grad(s.h, 0, None, 4, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    assert lib.lb_spgp_acq_grad(s.h, 0, _p(ap), 0, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    assert lib.lb_spgp_acq_grad(s.h, 0, _p(ap), 4, None, 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    for acq_id in (-1, 2, 7):
        assert lib.lb_spgp_acq_grad(s.h, acq_id, _p(ap), 4, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_ARG
    # before lb_spgp_compute: no data, then data without factors, then factors dropped by lb_spgp_set_data
    fresh = Raw()
    assert lib.lb_spgp_query_grad(fresh.h, 4, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_STATE
    assert lib.lb_spgp_acq_grad(fresh.h, 0, _p(ap), 4, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_STATE
    Xc = np.ascontiguousarray(X)
    yc = np.ascontiguousarray(y)
    assert lib.lb_spgp_set_data(fresh.h, Xc.shape[0], 3, _p(Xc), _p(yc)) == 0
    assert lib.lb_spgp_query_grad(fresh.h, 4, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_STATE
    assert lib.lb_spgp_acq_grad(fresh.h, 1, _p(ap), 4, _p(Xq), 1, None, 0.0, None, _p(v), _p(o)) == LB_ERR_STATE
    assert lib.lb_spgp_set_data(s.h, Xc.shape[0], 3, _p(Xc), _p(yc)) == 0
    assert lib.lb_spgp_query_grad(s.h, 4, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_STATE
    # a likelihood evaluation replaces the factors: no queries until the next compute, whose b1 is fresh
    w2 = np.ascontiguousarray(w)
    assert lib.lb_spgp_compute(s.h, M, w2.size, _p(w2), JITTER) == 0
    before = s.query_grad(Xq)
    f = C.c_double()
    w3 = np.ascontiguousarray(w + 0.01)
    assert lib.lb_spgp_lik(s.h, M, w3.size, _p(w3), JITTER, C.addressof(f), None) == 0
    assert lib.lb_spgp_query_grad(s.h, 4, _p(Xq), 1, None, None, _p(o), None) == LB_ERR_STATE
    assert lib.lb_spgp_compute(s.h, M, w3.size, _p(w3), JITTER) == 0
    st3 = O.State(w3, X, y, M, JITTER)
    _, _, dmu3, _ = s.query_grad(Xq)
    _, _, dmo, _, mag = SG.query_grad(st3, Xq)
    assert np.all(np.abs(dmu3 - dmo) <= BOUND * mag)
    assert lib.lb_spgp_compute(s.h, M, w2.size, _p(w2), JITTER) == 0
    assert all(np.array_equal(p, q) for p, q in zip(before, s.query_grad(Xq)))


class _Linear:
    """an input-dependent mean: m(x) = a . x + 0.3, with its input gradient"""
    A = np.array([0.4, -0.7])

    def __init__(self, params=None, dim_out=1):
        self._dim_out = dim_out

    def h_params_size(self):
        return 0

    def h_params(self):
        return np.zeros(0)

    def set_h_params(self, p):
        pass

    def grad(self, x, gp):
        return np.zeros((self._dim_out, 0))

    def is_constant(self):
        return False

    def __call__(self, v, gp):
        return np.full(self._dim_out, float(np.dot(self.A, np.asarray(v)[:2])) + 0.3)

    def batch(self, xs, gp):
        return np.stack([self(x, gp) for x in np.atleast_2d(xs)], axis=0)

    def grad_x(self, xs, gp):
        xs = np.atleast_2d(xs)
        g = np.zeros((xs.shape[0], self._dim_out, xs.shape[1]))
        g[:, :, :2] = self.A
        return g


class _OptParams:
    class acqui_ucb:
        alpha = 0.5

    class acqui_ei:
        jitter = 0.0

    class model_spgp:
        jitter = 1e-6
        samples_percent = 20
        min_m = 1

    class opt_rprop:
        iterations = 150
        eps_stop = 0.0

    class opt_batchedgradient:
        candidates = 2000
        starts = 16
        iterations = 300
        alpha = 0.01

    class opt_batchedrandom:
        candidates = 2000
        refinements = 2
        shrink = 0.1


def _fit_model(mean_cls=None, seed=12, N=60):
    from limbo_b200 import mean, model
    rng = np.random.default_rng(seed)
    X = rng.random((N, 2))
    Y = np.sin(5 * X[:, :1]) * np.cos(3 * X[:, 1:]) + 0.3 * X[:, :1]
    m = model.SPGP(params=_OptParams, mean=mean_cls or mean.Data, rng=np.random.default_rng(seed))
    m.compute(X, Y)
    mv = m.mean_function().batch(X, m)[:, 0]
    st = O.State(m.hyper_params(), X, Y[:, 0] - mv, m.nb_pseudo_samples(), JITTER)
    return m, st, X, Y


def test_input_dependent_mean_adds_its_gradient():
    from limbo_b200 import acqui, mean
    m, st, X, Y = _fit_model(mean.function_ard(_Linear), seed=3)
    Xq = np.ascontiguousarray(np.random.default_rng(4).random((50, 2)))
    mq = m.mean_function().batch(Xq, m)[:, 0]
    mu, s2, dmu, ds2 = m.query_grad_batch(Xq)
    mo, so, dmo, dso, mag = SG.query_grad(st, Xq)
    assert np.all(np.abs(mu[:, 0] - (mo + mq)) <= 1e-9 * st.c) and np.all(np.abs(s2 - so) <= 1e-9 * st.c)
    assert np.all(np.abs(dmu - (dmo + _Linear.A)) <= BOUND * mag + 1e-15) and np.all(np.abs(ds2 - dso) <= BOUND * mag)
    v, g = acqui.UCB(m, 0, params=_OptParams).grad_batch(Xq)
    rv, rg = AG.ucb(mo + mq, so, dmo + _Linear.A, dso, 0.5)
    assert np.allclose(v, rv, rtol=0, atol=1e-9) and np.allclose(g, rg, rtol=0, atol=1e-8)
    ap = np.array([0.5, 0.0])
    v0, g0 = m.acq_grad_batch(0, ap, Xq)
    assert np.array_equal(v0, v) and np.array_equal(g0, g)
    assert np.array_equal(m.acq_argmax_batch(0, ap, Xq, return_values=True)[2], v)
    # a mean without an input gradient: no silent zero
    m._mean_function.grad_x = lambda xs, gp: mean.BaseMean.grad_x(m._mean_function, xs, gp)
    with pytest.raises(NotImplementedError):
        m.acq_grad_batch(0, ap, Xq)
    with pytest.raises(NotImplementedError):
        m.query_grad_batch(Xq)


@pytest.mark.parametrize("acq_name", ["UCB", "EI"])
def test_gradient_search_reaches_the_lbfgsb_maximum(acq_name):
    from limbo_b200 import acqui, bayes_opt
    m, st, X, Y = _fit_model()
    acq = getattr(acqui, acq_name)(m, 0, params=_OptParams)
    Xq = np.ascontiguousarray(np.random.default_rng(1).random((64, 2)))
    v1, g1 = acq.grad_batch(Xq)
    ap = np.array([0.5, 0.0]) if acq_name == "UCB" else np.array([acq._f_max, 0.0])
    v2, g2 = m.acq_grad_batch(0 if acq_name == "UCB" else 1, ap, Xq)
    assert np.array_equal(v1, v2) and np.array_equal(g1, g2)
    ym = float(Y.mean())
    f_max = float((st.predict(X)[0] + ym).max())

    def neg(x):
        mu, s2, dmu, ds2, _ = SG.query_grad(st, np.atleast_2d(x))
        v, g = AG.ucb(mu + ym, s2, dmu, ds2, 0.5) if acq_name == "UCB" else AG.ei(mu + ym, s2, dmu, ds2, f_max, 0.0)
        return -float(v[0]), -g[0]
    rng = np.random.default_rng(2)
    starts = np.vstack([rng.random((40, 2)), np.stack(np.meshgrid(np.linspace(0.05, 0.95, 6), np.linspace(0.05, 0.95, 6)), -1).reshape(-1, 2)])
    best = max(-minimize(neg, s, jac=True, method="L-BFGS-B", bounds=[(0, 1), (0, 1)], options={"ftol": 1e-15, "gtol": 1e-12}).fun
               for s in starts)
    xg = bayes_opt.BatchedGradientSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    xr = bayes_opt.BatchedRandomSearch(_OptParams, np.random.default_rng(0))(acq, 2, True)
    vg, vr = acq.grad_batch(np.vstack([xg, xr]))[0]
    print(f"{acq_name}: gradient search {vg:.12f}, L-BFGS-B {best:.12f}, random search {vr:.12f}")
    assert vg >= best - 1e-6, (vg, best)
    assert vg >= vr


def test_cpp_spgp_grad_dropin():
    run_dropin("spgp_grad_dropin_test", "SPGP GRAD DROPIN OK")
