"""Multi-objective BO on the device: lb_ehvi_argmax (both models' queries on their own streams, ehvi_kernel and the block argmax)
against the reference's own acqui::Ehvi (tests/golden/ehvi), against the oracle's table form at N = 16384, every error code,
determinism and concurrency, lb_pareto_set against the oracle, and a bayes_opt.Ehvi run on mop2."""
import ctypes as C
import glob
import os
import threading
import time

import numpy as np
import pytest

from dropin import run_dropin
from oracle import ehvi as E

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ehvi")
GP_FIXTURES = [p for p in sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))) if "X" in np.load(p).files]
LB_ERR_ARG, LB_ERR_STATE, LB_ERR_UNSUPPORTED = -1, -3, -5


def _params(noise=0.01):
    class P:
        class kernel:
            pass
    P.kernel.noise = noise
    return P


def _pair(X, Y, noise=0.01, kernel="MaternFiveHalves", mean="Data"):
    from limbo_b200 import kernel as K, mean as Mn, model
    P = _params(noise)
    ms = [model.GP(X.shape[1], 1, params=P, kernel=getattr(K, kernel), mean=getattr(Mn, mean)) for _ in range(2)]
    for j, m in enumerate(ms):
        if len(X):
            m.compute(X, Y[:, j:j + 1])
    return ms


def _check_against_oracle(front, r, mu, s, vals, idx, tag):
    want, scale = E.ehvi2d_tables(front, r, mu[:, 0], s[:, 0], mu[:, 1], s[:, 1])
    tol = E.tolerance(want, scale)
    err = np.abs(vals - want)
    rel = err.max() / max(np.abs(want).max(), 1e-300)
    print(tag, "max |dev - oracle|", err.max(), "relative to the largest value", rel, "max err / tol", (err / np.maximum(tol, 1e-300)).max())
    assert np.all(err <= tol)
    # a plain bound beside the derived one: the largest measured on an H100 is 5.7e-9 (candidates on the samples, where
    # sigma^2 + noise ~ 1e-6 and the cells cancel); everywhere else it is below 1e-13
    assert rel <= 2e-8
    top = np.sort(want)[::-1]
    if idx != int(np.argmax(want)):  # only where the oracle's top two are closer than the tolerance
        assert top[0] - top[1] <= tol.max(), (tag, idx, int(np.argmax(want)))
    return want


@pytest.mark.parametrize("path", GP_FIXTURES, ids=os.path.basename)
def test_ehvi_matches_reference_fixtures(path):
    from limbo_b200 import acqui
    g = np.load(path)
    ms = _pair(g["X"], g["Y"], float(g["noise"]))
    for j, m in enumerate(ms):
        mu, s2 = m.query_batch(g["Xq"])
        assert np.abs(mu[:, 0] - g["mu"][:, j]).max() <= 1e-10 and np.abs(s2 - g["s"][:, j]).max() <= 1e-10
    best, idx, vals = acqui.EHVI(ms, g["front"], g["r"]).argmax_batch(g["Xq"], return_values=True)
    want = _check_against_oracle(g["front"], g["r"], g["mu"], g["s"], vals, idx, os.path.basename(path))
    assert np.abs(want - g["ehvi"]).max() <= 1e-13 * np.abs(g["ehvi"]).max()  # the oracle itself (tests/test_ehvi_host.py)
    assert idx == int(np.argmax(g["ehvi"])) and best == vals[idx]


def test_ehvi_prior_fixture():
    """Two models without samples score with their prior (mu = 0, sigma^2 + noise = 1.01): every value is equal, index 0 wins."""
    from limbo_b200 import acqui
    g = np.load(os.path.join(GOLDEN, "prior.npz"))
    ms = _pair(np.zeros((0, 2)), np.zeros((0, 2)))
    best, idx, vals = acqui.EHVI(ms, g["front"], g["r"]).argmax_batch(g["Xq"], return_values=True)
    _check_against_oracle(g["front"], g["r"], g["mu"], g["s"], vals, idx, "prior")
    assert np.all(vals == vals[0]) and idx == 0 and abs(vals[0] - g["ehvi"][0]) <= 1e-12 * g["ehvi"][0]


def _big_pair(N=16384, D=6):
    rng = np.random.default_rng(5)
    X = rng.random((N, D))
    Y = E.zdt2(X) + 0.01 * np.stack([np.sin(7 * X[:, 1]), np.cos(5 * X[:, 2])], axis=1)
    from limbo_b200 import kernel, mean, model
    ms = []
    for j in range(2):
        m = model.GP(D, 1, params=_params(), kernel=kernel.SquaredExpARD, mean=mean.Data)
        m.compute(X, Y[:, j:j + 1])
        ms.append(m)
    return ms, rng


@pytest.fixture(scope="module")
def big():
    return _big_pair()


@pytest.mark.parametrize("k", [16, 256, 4096])
def test_ehvi_against_oracle_n16384(big, k):
    """N = 16384, D = 6, M = 20000.  k = 16 and 256: the oracle scores every candidate.  k = 4096: the oracle's table form over
    all 20000 candidates (1.7e11 cells) would take hours on the host, so, as a deviation from checking the argmax over all M, it
    scores the device's 32 best and 256 random candidates; every value must be within tolerance and the device's argmax must be
    the oracle's argmax over that set.  A candidate the device undervalues outside that set is not caught at this k; the full
    comparisons at k = 16 and 256 run the same kernel code."""
    ms, rng = big
    M = 20000
    Xq = rng.random((M, 6))
    mus = [m.query_batch(Xq) for m in ms]
    mu = np.stack([mus[0][0][:, 0], mus[1][0][:, 0]], axis=1)
    s = np.stack([mus[0][1], mus[1][1]], axis=1)
    # a front around the models' predictions, so that EHVI is far from 0 on part of the candidates
    lo, hi = np.quantile(mu, 0.7, axis=0), mu.max(axis=0) + 0.3
    f0 = np.sort(rng.uniform(lo[0], hi[0], k))
    front = np.stack([f0, np.sort(rng.uniform(lo[1], hi[1], k))[::-1]], axis=1)[rng.permutation(k)]
    r = (float(mu[:, 0].min()) - 1.0, float(mu[:, 1].min()) - 1.0)
    t0 = time.perf_counter()
    best, idx, vals = ms[0].ehvi_argmax_batch(ms[1], r, front, Xq, return_values=True)
    print("k", k, "lb_ehvi_argmax", time.perf_counter() - t0, "s; share of positive values", (vals > 0).mean())
    assert best == vals[idx] and (vals > 0).sum() >= 10  # k = 16: 93 positive values (H100); 0 elsewhere, underflowed tails
    if k <= 256:
        _check_against_oracle(front, r, mu, s, vals, idx, f"k={k}")
    else:
        sub = np.unique(np.concatenate([np.argsort(-vals, kind="stable")[:32], rng.choice(M, 256, replace=False)]))
        want = _check_against_oracle(front, r, mu[sub], s[sub], vals[sub], int(np.flatnonzero(sub == idx)[0]), f"k={k} subset")
        assert sub[int(np.argmax(want))] == idx or np.sort(want)[-1] - np.sort(want)[-2] <= E.tolerance(want, 0 * want).max() + 1e-9


def test_ehvi_k0_and_repeat_bit_identical(big):
    ms, rng = big
    Xq = rng.random((3000, 6))
    mus = [m.query_batch(Xq) for m in ms]
    mu = np.stack([mus[0][0][:, 0], mus[1][0][:, 0]], axis=1)
    s = np.stack([mus[0][1], mus[1][1]], axis=1)
    r = (-2.0, -9.0)
    best, idx, vals = ms[0].ehvi_argmax_batch(ms[1], r, np.zeros((0, 2)), Xq, return_values=True)
    _check_against_oracle(np.zeros((0, 2)), r, mu, s, vals, idx, "k=0")
    front = np.stack([np.linspace(0, 1, 300), np.linspace(1, 0, 300) ** 2], axis=1)
    first = ms[0].ehvi_argmax_batch(ms[1], r, front, Xq, return_values=True)
    for _ in range(3):
        again = ms[0].ehvi_argmax_batch(ms[1], r, front[::-1].copy(), Xq, return_values=True)  # input order does not matter
        assert again[:2] == first[:2] and np.array_equal(again[2], first[2])


def test_ehvi_argument_errors(big):
    from limbo_b200 import _lib, kernel, mean, model
    lib = _lib.load()
    ms, rng = big
    Xq = np.ascontiguousarray(rng.random((100, 6)))
    best, idx = C.c_double(), C.c_int64()
    r = np.array([-5.0, -5.0])
    F = np.ascontiguousarray(rng.random((10, 2)))

    def call(a, b, rr=r, k=10, f=F, M=100, x=Xq, bv=True, bi=True):
        return lib.lb_ehvi_argmax(a, b, rr.ctypes.data if rr is not None else None, k, f.ctypes.data if f is not None else None, M,
                                  x.ctypes.data, None, 0.0, None, 0.0, None, C.addressof(best) if bv else None,
                                  C.addressof(idx) if bi else None)
    h0, h1 = ms[0]._h, ms[1]._h
    assert call(h0, h1) == 0
    assert call(h0, h0) == LB_ERR_ARG
    assert call(h0, None) == LB_ERR_ARG
    assert call(h0, h1, M=0) == LB_ERR_ARG and call(h0, h1, M=-3) == LB_ERR_ARG
    assert call(h0, h1, rr=None) == LB_ERR_ARG and call(h0, h1, f=None) == LB_ERR_ARG and call(h0, h1, k=-1) == LB_ERR_ARG
    assert call(h0, h1, bv=False) == LB_ERR_ARG and call(h0, h1, bi=False) == LB_ERR_ARG
    for bad in (np.nan, np.inf, -np.inf):
        fb = F.copy()
        fb[3, 1] = bad
        rb = r.copy()
        rb[0] = bad
        assert call(h0, h1, f=fb) == LB_ERR_ARG and call(h0, h1, rr=rb) == LB_ERR_ARG
    big_front = np.ascontiguousarray(rng.random((_lib.EHVI_MAX_K + 1, 2)))
    assert call(h0, h1, k=_lib.EHVI_MAX_K + 1, f=big_front) == LB_ERR_UNSUPPORTED
    other = model.GP(3, 1, params=_params(), kernel=kernel.MaternFiveHalves, mean=mean.Data)  # D = 3 against D = 6
    other.compute(rng.random((20, 3)), rng.random((20, 1)))
    assert call(h0, other._h) == LB_ERR_ARG
    fresh = model.GP(6, 1)  # no kernel state on the device yet
    assert call(h0, fresh._h) == LB_ERR_STATE


def test_ehvi_dev_equals_host(big):
    import torch
    from limbo_b200 import _lib
    lib = _lib.load()
    ms, rng = big
    Xq = rng.random((2500, 6))
    F = np.ascontiguousarray(np.stack([np.linspace(0, 1, 40), np.linspace(1, 0, 40)], axis=1))
    r = np.array([-1.0, -1.0])
    ref = ms[0].ehvi_argmax_batch(ms[1], r, F, Xq, return_values=True)
    means = [torch.from_numpy(np.ascontiguousarray(m.mean_function().batch(Xq, m)[:, 0])).cuda() for m in ms]
    dXq = torch.from_numpy(Xq).cuda()
    dacq = torch.empty(len(Xq), dtype=torch.float64, device="cuda")
    dbest = torch.empty(1, dtype=torch.float64, device="cuda")
    didx = torch.empty(1, dtype=torch.int64, device="cuda")
    rc = lib.lb_ehvi_argmax_dev(ms[0]._h, ms[1]._h, r.ctypes.data, 40, F.ctypes.data, len(Xq), dXq.data_ptr(), means[0].data_ptr(), 0.0,
                                means[1].data_ptr(), 0.0, dacq.data_ptr(), dbest.data_ptr(), didx.data_ptr())
    assert rc == 0 and lib.lb_sync(ms[0]._h) == 0
    assert float(dbest.item()) == ref[0] and int(didx.item()) == ref[1]
    assert np.array_equal(dacq.cpu().numpy(), ref[2])


def test_ehvi_threads_with_swapped_pairs():
    """Two threads score (a, b) and (b, a) 20 times each while a third queries b: the locks keep them deadlock-free and every
    result equals the serial one."""
    rng = np.random.default_rng(11)
    X = rng.random((400, 3))
    a, b = _pair(X, E.zdt2(X))
    Xq = rng.random((3000, 3))
    F = np.stack([np.linspace(0, 1, 50), np.linspace(1, 0, 50)], axis=1)
    r_ab = a.ehvi_argmax_batch(b, (-1, -1), F, Xq, return_values=True)
    r_ba = b.ehvi_argmax_batch(a, (-1, -1), F, Xq, return_values=True)
    q_b = b.query_batch(Xq)
    errors = []

    def loop(fn):
        try:
            for _ in range(20):
                fn()
        except Exception as e:  # reported below
            errors.append(repr(e))

    def ab():
        r = a.ehvi_argmax_batch(b, (-1, -1), F, Xq, return_values=True)
        if r[:2] != r_ab[:2] or not np.array_equal(r[2], r_ab[2]):
            errors.append("a,b differs")

    def ba():
        r = b.ehvi_argmax_batch(a, (-1, -1), F, Xq, return_values=True)
        if r[:2] != r_ba[:2] or not np.array_equal(r[2], r_ba[2]):
            errors.append("b,a differs")

    def qb():
        m, s = b.query_batch(Xq)
        if not (np.array_equal(m, q_b[0]) and np.array_equal(s, q_b[1])):
            errors.append("lb_query on b differs")

    th = [threading.Thread(target=loop, args=(f,), daemon=True) for f in (ab, ba, qb)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in th), "a thread did not finish"
    assert not errors, errors


@pytest.mark.parametrize("K", [2, 3])
def test_pareto_set_against_oracle_n16384(K):
    from limbo_b200 import pareto
    rng = np.random.default_rng(K)
    n = 16384
    O = np.round(rng.normal(size=(n, K)), 2)  # coarse grid: exact ties and duplicates on the front
    O[-200:] = O[np.argsort(-O[:, 0])[:200]]  # duplicates of the best points
    got = pareto.pareto_set_indices(O)
    want = E.pareto_set(O)
    print("K", K, "front", len(want))
    assert np.array_equal(got, want)  # same ascending-index rule for ties
    assert len(set(map(tuple, O[want]))) < len(want)  # duplicates really are on the front


def test_pareto_set_errors_and_tuples():
    from limbo_b200 import _lib, pareto
    lib = _lib.load()
    h = pareto._handle(0)
    O = np.ascontiguousarray(np.random.default_rng(0).random((50, 2)))
    idx, nf = np.empty(50, dtype=np.int64), C.c_int64()
    bad = O.copy()
    bad[7, 0] = np.nan
    assert lib.lb_pareto_set(h, 50, 2, bad.ctypes.data, idx.ctypes.data, C.addressof(nf)) == LB_ERR_ARG
    wide = np.ascontiguousarray(np.random.default_rng(1).random((10, _lib.PARETO_MAX_K + 1)))
    assert lib.lb_pareto_set(h, 10, _lib.PARETO_MAX_K + 1, wide.ctypes.data, idx.ctypes.data, C.addressof(nf)) == LB_ERR_UNSUPPORTED
    assert lib.lb_pareto_set(h, 50, 0, O.ctypes.data, idx.ctypes.data, C.addressof(nf)) == LB_ERR_ARG
    pts = [(np.array([float(i)]), O[i], np.zeros(2)) for i in range(50)]
    front = pareto.pareto_set(pts, 1)
    assert [int(p[0][0]) for p in front] == list(E.pareto_set(O))


def test_bayes_opt_ehvi_on_mop2():
    """30 iterations on mop2 (D = 2) from 10 random samples: the data front's hypervolume above (-11, -11) beats that of 40
    uniform random samples by more than 1.  Measured on an H100 (700 W) with these seeds: 143.32 against 140.93 (the square
    from the reference point to the origin alone is 121).  The loop's models are refitted from scratch each iteration (BoMulti._update_models)."""
    from limbo_b200 import bayes_opt

    class P:
        class kernel:
            noise = 1e-6

        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 30

    r = (-11.0, -11.0)
    bo = bayes_opt.Ehvi(params=P, rng=np.random.default_rng(0))
    bo.optimize(lambda x: E.mop2(x)[0], 2)
    Y = np.stack(bo.observations())
    assert Y.shape == (40, 2) and len(bo.models()) == 2 and bo.pareto_model() == []
    bo.update_pareto_data()
    front = np.stack([p[1] for p in bo.pareto_data()])
    hv = E.hypervolume(front, r)
    Yr = E.mop2(np.random.default_rng(1).random((40, 2)))
    hv_rand = E.hypervolume(Yr, r)
    print("hypervolume: ehvi", hv, "random", hv_rand, "front size", len(front))
    assert np.array_equal(front, Y[E.pareto_set(Y)])
    assert hv > hv_rand + 1.0


def test_cpp_ehvi_dropin():
    """The reference's primary acqui::Ehvi over reference GPs against the specialisation over limbo_b200::model::GP, one point
    at a time, answering a BatchRequest, and driven by BatchedRandom (tests/cpp/ehvi_dropin_test.cpp)."""
    run_dropin("ehvi_dropin_test", "EHVI DROPIN OK")
