"""The sparsified model on the device: lb_sparsify (limbo_b200/csrc/sparsify.cu) against the reference's own _sparsify
(tests/golden/sparsify) and against the oracle beyond the fixtures, its error codes, and model.SparsifiedGP, MultiGP over it,
BOptimizer over it and the compiled C++ drop-in against the reference's SparsifiedGP."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np
import pytest

from oracle import sparsify as oracle_sparsify

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "sparsify", "*.npz")))
LB_ERR_ARG, LB_ERR_UNSUPPORTED = -1, -5


@pytest.fixture(scope="module")
def gp():
    from limbo_b200 import model
    return model.GP(1, 1)


def _call(h, X, max_points):
    """lb_sparsify; returns (rc, kept, removed, removed_score)"""
    from limbo_b200 import _lib
    X = np.ascontiguousarray(X, dtype=np.float64)
    N, D = X.shape
    kept = np.full(N, -7, dtype=np.int64)
    removed = np.full(max(N, 1), -7, dtype=np.int64)
    score = np.full(max(N, 1), np.nan)
    nk = C.c_int64(-1)
    rc = _lib.load().lb_sparsify(h, N, D, X.ctypes.data, max_points, kept.ctypes.data, C.addressof(nk), removed.ctypes.data,
                                 score.ctypes.data)
    nr = N - nk.value
    return rc, kept[:nk.value], removed[:nr], score[:nr]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_sparsify_matches_reference_fixtures(gp, path):
    g = np.load(path)
    before = gp.launch_count()
    rc, kept, removed, score = _call(gp._h, g["X"], int(g["max_points"]))
    assert rc == 0
    assert np.array_equal(kept, g["kept"])
    assert np.array_equal(removed, g["removed"])
    assert np.array_equal(_bits(score), _bits(g["removed_score"]))
    if len(g["X"]) <= int(g["max_points"]):
        assert gp.launch_count() == before  # nothing launched


@pytest.mark.parametrize("seed,N,D,max_points", [(11, 3000, 1, 1000), (12, 4000, 6, 1500), (13, 2500, 12, 600), (14, 1000, 6, 6),
                                                 (15, 16384, 6, 4096)])
def test_sparsify_matches_oracle(gp, seed, N, D, max_points):
    X = np.random.default_rng(seed).uniform(-1.0, 1.0, (N, D))
    rc, kept, removed, score = _call(gp._h, X, max_points)
    assert rc == 0
    ok, orm, osc = oracle_sparsify.sparsify(X, max_points)
    assert np.array_equal(kept, ok)
    assert np.array_equal(removed, orm)
    assert np.array_equal(_bits(score), _bits(osc))


def test_sparsify_lattice_ties(gp):
    X = np.stack(np.meshgrid(np.arange(40.0), np.arange(40.0), indexing="ij"), -1).reshape(-1, 2)
    rc, kept, removed, score = _call(gp._h, X, 300)
    assert rc == 0
    ok, orm, osc = oracle_sparsify.sparsify(X, 300)
    assert np.array_equal(removed, orm) and np.array_equal(kept, ok) and np.array_equal(_bits(score), _bits(osc))


def test_sparsify_dev_equals_host(gp):
    import torch
    from limbo_b200 import _lib
    X = np.random.default_rng(21).normal(size=(5000, 4))
    rc, kept, removed, score = _call(gp._h, X, 1200)
    assert rc == 0
    dX = torch.from_numpy(X).cuda()
    dk = torch.full((5000,), -7, dtype=torch.int64, device="cuda")
    dr = torch.full((5000,), -7, dtype=torch.int64, device="cuda")
    ds = torch.zeros(5000, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    nk = C.c_int64(-1)
    rc = _lib.load().lb_sparsify_dev(gp._h, 5000, 4, dX.data_ptr(), 1200, dk.data_ptr(), C.addressof(nk), dr.data_ptr(), ds.data_ptr())
    assert rc == 0 and nk.value == 1200
    assert np.array_equal(dk[:1200].cpu().numpy(), kept)
    assert np.array_equal(dr[:3800].cpu().numpy(), removed)
    assert np.array_equal(_bits(ds[:3800].cpu().numpy()), _bits(score))


def test_sparsify_error_codes(gp):
    X = np.random.default_rng(3).normal(size=(200, 6))
    before = gp.launch_count()
    assert _call(gp._h, X, 5)[0] == LB_ERR_ARG  # max_points < D
    assert _call(gp._h, np.random.default_rng(3).normal(size=(200, 65)), 100)[0] == LB_ERR_UNSUPPORTED  # D > 64
    assert gp.launch_count() == before
    Xn = X.copy()
    Xn[17, 3] = np.nan
    assert _call(gp._h, Xn, 100)[0] == LB_ERR_ARG
    Xi = X.copy()
    Xi[5, 0] = np.inf
    assert _call(gp._h, Xi, 100)[0] == LB_ERR_ARG
    rc, kept, removed, _ = _call(gp._h, X, 100)  # the handle still works after the errors
    assert rc == 0 and np.array_equal(kept, oracle_sparsify.sparsify(X, 100)[0])


def _P(max_points, **sections):
    class P:
        class model_sparse_gp:
            pass
    P.model_sparse_gp.max_points = max_points
    for name, attrs in sections.items():
        setattr(P, name, type(name, (), attrs))
    return P


def test_sparsified_gp_compute_is_gp_on_kept_subset():
    from limbo_b200 import model
    from oracle import oracle as O
    rng = np.random.default_rng(5)
    X = rng.uniform(0.0, 1.0, (900, 3))
    y = np.sin(3 * X).sum(1)[:, None]
    Xq = rng.uniform(0.0, 1.0, (300, 3))
    P = _P(400)
    sgp = model.SparsifiedGP(params=P)
    sgp.compute(list(X), list(y))
    kept = oracle_sparsify.sparsify(X, 400)[0]
    assert sgp.nb_samples() == 400 and np.array_equal(np.stack(sgp.samples()), X[kept])
    ref = model.GP(params=P)  # the same defaults: MaternFiveHalves, mean::Data
    ref.compute(X[kept], y[kept])
    mu, s2 = sgp.query_batch(Xq)
    mu_r, s2_r = ref.query_batch(Xq)
    assert np.array_equal(_bits(mu), _bits(mu_r)) and np.array_equal(_bits(s2), _bits(s2_r))
    assert sgp.compute_log_lik() == ref.compute_log_lik()
    og = O.OracleGP()  # mean::Data: the mean of the kept observations
    yk = y[kept]
    og.set_data(X[kept], yk - yk.mean())
    og.set_kernel(O.K_MATERN52, np.zeros(2), 0.01)
    og.fit()
    mu_o, s2_o = og.query(Xq)
    assert np.abs(mu - (mu_o + yk.mean())).max() < 1e-10 and np.abs(s2 - s2_o).max() < 1e-10
    c = sgp.copy()
    assert type(c) is model.SparsifiedGP


def test_sparsified_gp_add_sample():
    from limbo_b200 import model
    rng = np.random.default_rng(8)
    X = rng.uniform(0.0, 1.0, (60, 2))
    y = X.sum(1)
    sgp = model.SparsifiedGP(params=_P(50))
    sgp.compute(X[:40], y[:40, None])
    n0 = sgp.append_count()
    for i in range(40, 50):  # up to max_points: the incremental path
        sgp.add_sample(X[i], [y[i]])
    assert sgp.append_count() == n0 + 10 and sgp.nb_samples() == 50
    for i in range(50, 60):  # past it: re-sparsify max_points + 1 samples, exactly the oracle's removal
        before, yb = np.stack(sgp.samples()), sgp.observations_matrix()[:, 0].copy()
        sgp.add_sample(X[i], [y[i]])
        full, yfull = np.vstack([before, X[i]]), np.append(yb, y[i])
        kept, removed, _ = oracle_sparsify.sparsify(full, 50)
        assert len(removed) == 1 and sgp.nb_samples() == 50
        assert np.array_equal(np.stack(sgp.samples()), full[kept])
        assert np.array_equal(sgp.observations_matrix()[:, 0], yfull[kept])


def _accuracy_failures(multi: bool, seeds=20):
    """test_gp.cpp:815-905 (test_sparse_gp_accuracy) and :991-1080 (test_sparse_multi_gp), learned points only"""
    from limbo_b200 import kernel, mean, model
    P = _P(50, mean_constant={"constant": 1.0}, opt_rprop={"iterations": 300, "eps_stop": 0.0})
    fails = 0
    for seed in range(seeds):
        rng = np.random.default_rng(1000 + seed)
        X = rng.uniform(-2.0, 2.0, (100, 1))
        y = np.cos(X)
        if multi:
            g = model.MultiGP(params=P, kernel=kernel.SquaredExpARD, mean=mean.Constant,
                              hp_opt=model.ParallelLFOpt(P, inner=model.KernelLFOpt))
            s = model.MultiGP(params=P, kernel=kernel.SquaredExpARD, mean=mean.Constant,
                              hp_opt=model.ParallelLFOpt(P, inner=model.KernelLFOpt), gp_class=model.SparsifiedGP)
        else:
            g = model.GP(params=P, kernel=kernel.SquaredExpARD, mean=mean.Constant, hp_opt=model.KernelLFOpt(P))
            s = model.SparsifiedGP(params=P, kernel=kernel.SquaredExpARD, mean=mean.Constant, hp_opt=model.KernelLFOpt(P))
        for m in (g, s):
            m.compute(X, y, False)
            m.optimize_hyperparams()
        mu_g, s2_g = g.query_batch(X)
        mu_s, s2_s = s.query_batch(X)
        if multi:
            assert s.gp_models()[0].nb_samples() == 50
        else:
            assert s.nb_samples() == 50
        fails += bool(np.abs(mu_g - mu_s).max() > 1e-2 or np.abs(s2_g - s2_s).max() > 1e-2)
    return fails


def test_sparse_gp_accuracy():
    assert _accuracy_failures(False) / 20 < 0.1


def test_sparse_multi_gp_accuracy():
    assert _accuracy_failures(True) / 20 < 0.1


def test_boptimizer_with_sparsified_gp():
    from limbo_b200 import acqui, bayes_opt, kernel, mean, model
    P = _P(25, kernel={"noise": 1e-6}, kernel_maternfivehalves={"sigma_sq": 1.0, "l": 0.3}, init_randomsampling={"samples": 10},
           stop_maxiterations={"iterations": 30}, opt_batchedrandom={"candidates": 20000, "refinements": 2, "shrink": 0.1},
           acqui_ucb={"alpha": 0.2})
    sol = np.array([0.25, 0.75])

    def f(x):
        return -float(((x - sol) ** 2).sum())
    sgp = model.SparsifiedGP(2, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    bo = bayes_opt.BOptimizer(sgp, params=P, acqui=acqui.UCB, rng=np.random.default_rng(0))
    bo.optimize(f, 2)
    assert len(bo.samples()) == 40 and sgp.nb_samples() == 25
    assert ((bo.best_sample() - sol) ** 2).sum() < 1e-2


def test_cpp_sparsified_dropin():
    binary = os.path.join(ROOT, "oracle", "_ref", "sparse_dropin_test")
    if not os.path.exists(binary):
        pytest.skip("oracle/_ref/sparse_dropin_test not built (needs the reference's sources at build time)")
    r = subprocess.run([binary], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "SPARSE DROPIN OK" in r.stdout, r.stdout + r.stderr
