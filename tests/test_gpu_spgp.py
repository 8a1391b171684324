"""The pseudo-input sparse GP on the device (lb_spgp_*, limbo_b200/csrc/spgp.cu) against the NumPy restatement of the reference's
experimental::model::SPGP (oracle/spgp.py): likelihood, gradient, _compute + _predict and the acquisition argmax up to
N = 16384, M = 1638, D = 6; central differences of the device value; the error codes; and model.SPGP through compute, query and
BOptimizer."""
import ctypes as C
import glob
import math
import os

import numpy as np
import pytest

from dropin import run_dropin
from oracle import spgp as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "spgp", "*.npz")))
LB_ERR_ARG, LB_ERR_STATE, LB_ERR_UNSUPPORTED = -1, -3, -5
JITTER = 1e-6


class Raw:
    """lb_spgp handle over the raw ABI."""

    def __init__(self):
        from limbo_b200 import _lib
        self.lib = _lib.load()
        self.h = C.c_void_p()
        assert self.lib.lb_spgp_create(C.byref(self.h), 0) == 0

    def __del__(self):
        self.lib.lb_spgp_destroy(self.h)

    def set_data(self, X, y):
        X = np.ascontiguousarray(X, dtype=np.float64)
        y = np.ascontiguousarray(y, dtype=np.float64)
        return self.lib.lb_spgp_set_data(self.h, X.shape[0], X.shape[1], X.ctypes.data, y.ctypes.data)

    def lik(self, M, w, jitter=JITTER, grad=True, n_w=None):
        w = np.ascontiguousarray(w, dtype=np.float64)
        f = C.c_double(np.nan)
        g = np.full(w.size, np.nan) if grad else None
        rc = self.lib.lb_spgp_lik(self.h, M, w.size if n_w is None else n_w, w.ctypes.data, jitter, C.addressof(f),
                                  g.ctypes.data if grad else None)
        return rc, f.value, g

    def compute(self, M, w, jitter=JITTER):
        w = np.ascontiguousarray(w, dtype=np.float64)
        return self.lib.lb_spgp_compute(self.h, M, w.size, w.ctypes.data, jitter)

    def query(self, Xq, optimized=1):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        mu, s2 = np.full(len(Xq), np.nan), np.full(len(Xq), np.nan)
        rc = self.lib.lb_spgp_query(self.h, len(Xq), Xq.ctypes.data, optimized, mu.ctypes.data, s2.ctypes.data)
        return rc, mu, s2

    def ucb_argmax(self, Xq, alpha, optimized=1):
        Xq = np.ascontiguousarray(Xq, dtype=np.float64)
        ap = np.array([alpha, 0.0])
        best, idx = C.c_double(), C.c_int64(-1)
        rc = self.lib.lb_spgp_acq_argmax(self.h, 0, ap.ctypes.data, len(Xq), Xq.ctypes.data, optimized, None, 0.0, None,
                                         C.addressof(best), C.addressof(idx))
        return rc, best.value, idx.value


def _case(seed, N, D, hartmann=False):
    from limbo_b200 import synth
    rng = np.random.default_rng(seed)
    if hartmann:
        X = synth.points(seed, N, D)
        y = synth.targets(X)
    elif D == 1:
        X = rng.random((N, 1)) * 6.0
        y = np.cos(X[:, 0]) + 0.05 * rng.normal(size=N)
    else:
        X = rng.random((N, D))
        y = np.sin(3.0 * X).sum(axis=1) + 0.05 * rng.normal(size=N)
    y = y - y.mean()
    M = O.n_pseudo(N)
    w = O.init_w(X, y, M, rng.permutation(N))
    w = w + rng.normal(0.0, 0.05, w.size)  # away from the start, where pseudo-inputs coincide with samples
    Xq = rng.random((500, D)) * (6.0 if D == 1 else 1.0)
    return X, y, M, w, Xq


CASES = [(1, 100, 1, False), (2, 40, 2, False), (3, 41, 2, False), (4, 5, 2, False), (5, 300, 3, False), (6, 2000, 6, True),
         (7, 16384, 6, True)]


@pytest.mark.parametrize("seed,N,D,hartmann", CASES)
def test_parity_with_oracle(seed, N, D, hartmann):
    X, y, M, w, Xq = _case(seed, N, D, hartmann)
    s = Raw()
    assert s.set_data(X, y) == 0
    rc, f, g = s.lik(M, w)
    assert rc == 0
    fo, go = O.likelihood(w, X, y, M, JITTER)
    gerr = np.abs(g - go).max() / np.abs(go).max()
    print(f"N={N} M={M} D={D}: |df|/|f| = {abs(f - fo) / abs(fo):.2e}, |dg|/|g|inf = {gerr:.2e}")
    assert abs(f - fo) <= 1e-10 * abs(fo)
    assert gerr <= 1e-7
    rc0, f0, _ = s.lik(M, w, grad=False)
    assert rc0 == 0 and abs(f0 - f) <= 1e-12 * abs(f)
    assert s.compute(M, w) == 0
    st = O.State(w, X, y, M, JITTER)
    rc, mu, s2 = s.query(Xq)
    assert rc == 0
    mo, so = st.predict(Xq)
    print(f"  |dmu|/c = {np.abs(mu - mo).max() / st.c:.2e}, |ds2|/c = {np.abs(s2 - so).max() / st.c:.2e}")
    assert np.abs(mu - mo).max() <= 1e-9 * st.c
    assert np.abs(s2 - so).max() <= 1e-9 * st.c
    rc, best, idx = s.ucb_argmax(Xq, 0.5)
    assert rc == 0
    u = O.ucb(mo, so, 0.5)
    assert idx == int(np.argmax(u)), (idx, int(np.argmax(u)))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_parity_with_reference_fixtures(path):
    """The device against the reference's own SPGP (tests/golden/spgp, oracle/ref_shim/spgp_driver.cpp)."""
    g = np.load(path)
    X, y, M, w, jit, Xq = g["X"], g["y"], int(g["M"]), g["w"], float(g["jitter"]), g["Xq"]
    s = Raw()
    assert s.set_data(X, y - y.mean()) == 0
    rc, f, grad = s.lik(M, w, jitter=jit)
    assert rc == 0
    print(f"{os.path.basename(path)}: |df|/|f| = {abs(f - g['f']) / abs(g['f']):.2e}, "
          f"|dg|/|g|inf = {np.abs(grad - g['grad']).max() / np.abs(g['grad']).max():.2e}")
    assert abs(f - g["f"]) <= 1e-10 * abs(g["f"])
    assert np.abs(grad - g["grad"]).max() <= 1e-7 * np.abs(g["grad"]).max()
    assert s.compute(M, w, jitter=jit) == 0
    rc, mu, s2 = s.query(Xq)
    assert rc == 0
    c = O.unpack(w, M, X.shape[1])[2]
    mu_ref = g["mu"] - y.mean()
    assert np.abs(mu - mu_ref).max() <= 1e-9 * c
    assert np.abs(s2 - g["s2"]).max() <= 1e-9 * c
    rc, _, idx = s.ucb_argmax(Xq, 0.5)
    assert rc == 0 and idx == int(np.argmax(O.ucb(mu_ref, g["s2"], 0.5)))


def test_value_keeps_integer_division():
    X, y, M, w, _ = _case(3, 41, 2)  # N - M = 37
    s = Raw()
    s.set_data(X, y)
    _, f, _ = s.lik(M, w, grad=False)
    ff, _ = O.likelihood(w, X, y, M, JITTER, grad=False, fix_integer_division=True)
    sig = O.unpack(w, M, 2)[3]
    assert abs((f - ff) - 0.5 * math.log(sig)) <= 1e-9 * abs(ff)


def test_gradient_matches_central_differences():
    X, y, M, w, _ = _case(2, 40, 2)  # N - M = 36, even
    s = Raw()
    s.set_data(X, y)
    _, _, g = s.lik(M, w)
    h = 1e-6
    fd = np.empty(w.size)
    for i in range(w.size):
        e = np.zeros(w.size)
        e[i] = h
        fd[i] = (s.lik(M, w + e, grad=False)[1] - s.lik(M, w - e, grad=False)[1]) / (2 * h)
    assert np.abs(fd - g).max() <= 1e-6 * np.abs(g).max(), np.abs(fd - g).max() / np.abs(g).max()


def test_error_codes():
    X, y, M, w, Xq = _case(2, 40, 2)
    s = Raw()
    assert s.lik(M, w)[0] == LB_ERR_STATE  # no data
    assert s.set_data(np.zeros((10, 65)), np.zeros(10)) == LB_ERR_UNSUPPORTED
    Xn = X.copy()
    Xn[3, 1] = np.nan
    assert s.set_data(Xn, y) == LB_ERR_ARG
    yn = y.copy()
    yn[0] = np.inf
    assert s.set_data(X, yn) == LB_ERR_ARG
    assert s.set_data(X, y) == 0
    assert s.query(Xq)[0] == LB_ERR_STATE  # nothing computed yet
    assert s.lik(0, w[:2 * 1 + 2 + 2 * 0])[0] == LB_ERR_ARG  # M < 1
    wbig = np.zeros((41 + 1) * 2 + 2)
    assert s.lik(41, wbig)[0] == LB_ERR_ARG  # M > N
    assert s.lik(M, w, n_w=w.size - 1)[0] == LB_ERR_ARG
    wn = w.copy()
    wn[5] = np.nan
    assert s.lik(M, wn)[0] == LB_ERR_ARG
    c = O.unpack(w, M, 2)[2]
    assert s.lik(M, w, jitter=-2.0 * c)[0] == 1  # Q(0, 0) = c + jitter < 0: pivot 1
    assert s.compute(M, w, jitter=-2.0 * c) == 1
    assert s.query(Xq)[0] == LB_ERR_STATE
    assert s.lik(M, w)[0] == 0  # the handle recovers


def test_optimized_offset_and_prior():
    X, y, M, w, Xq = _case(5, 300, 3)
    s = Raw()
    s.set_data(X, y)
    assert s.compute(M, w) == 0
    _, mu1, s1 = s.query(Xq, optimized=1)
    _, mu0, s0 = s.query(Xq, optimized=0)
    sig = O.unpack(w, M, 3)[3]
    assert np.array_equal(mu1, mu0)
    assert np.abs((s1 - s0) - sig).max() <= 1e-15 * max(1.0, sig) * 4
    from limbo_b200 import kernel, model
    m = model.SPGP(3, 1, kernel=kernel.SquaredExpARD)
    mu, s2 = m.query_batch(Xq[:7])
    assert np.array_equal(mu, np.zeros((7, 1))) and np.array_equal(s2, np.full(7, m.kernel_function().sigma_sq()))


def test_spgp_fits_cos():
    from limbo_b200 import model
    rng = np.random.default_rng(11)
    X = rng.random((100, 1)) * 6.0
    y = np.cos(X[:, 0])
    m = model.SPGP(rng=np.random.default_rng(0))
    m.compute(X, y[:, None])
    assert m.nb_samples() == 100 and m.nb_pseudo_samples() == 10 and len(m.pseudo_samples()) == 10
    mu, s2 = m.query_batch(X)
    rmse = float(np.sqrt(np.mean((mu[:, 0] - y) ** 2)))
    print("rmse", rmse, "std", y.std())
    assert rmse < y.std()
    assert np.all(s2 > 0)
    # the model's factors are the oracle's at the optimum it found
    st = O.State(m.hyper_params(), X, y - y.mean(), 10, JITTER)
    mo, so = st.predict(X)
    assert np.abs(mu[:, 0] - (mo + y.mean())).max() <= 1e-9 * st.c
    assert np.abs(s2 - so).max() <= 1e-9 * st.c


def test_boptimizer_with_spgp():
    from limbo_b200 import acqui, bayes_opt, model

    class P:
        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 15

        class model_spgp:
            jitter = 1e-6
            samples_percent = 50
            min_m = 1

        class opt_batchedrandom:
            candidates = 5000
            refinements = 1
            shrink = 0.1

        class opt_rprop:
            iterations = 100
            eps_stop = 0.0

    sol = np.array([0.25, 0.75])

    def f(x):
        return -float(((x - sol) ** 2).sum())
    m = model.SPGP(params=P, rng=np.random.default_rng(1))
    bo = bayes_opt.BOptimizer(m, params=P, acqui=acqui.UCB, rng=np.random.default_rng(0))
    bo.optimize(f, 2)
    obs = [float(o[0]) for o in bo.observations()]
    assert len(obs) == 25 and m.nb_samples() == 25 and m.nb_pseudo_samples() == 12
    assert max(obs[10:]) > max(obs[:10]), (max(obs[10:]), max(obs[:10]))


def test_cpp_spgp_dropin():
    run_dropin("spgp_dropin_test", "SPGP DROPIN OK")
