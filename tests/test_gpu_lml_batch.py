"""lb_lml_grad_batch / GP.lml_grad_batch and KernelLFOpt over BatchedParallelRepeater on the device: every row against the single
path (lb_set_kernel + lb_fit + lb_log_lik + lb_kernel_grad_log_lik on a copy of the GP) and the oracle, determinism across batch
sizes and positions, non-positive pivots, the model state, the launch count, the error codes, concurrent use, and the optimiser
against ParallelRepeater(Rprop)."""
import ctypes as C
import math
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dropin import run_dropin  # noqa: E402
from limbo_b200 import _lib, kernel, mean, model, opt, synth  # noqa: E402

KERNELS = {0: kernel.SquaredExpARD, 1: kernel.MaternFiveHalves, 2: kernel.MaternThreeHalves, 3: kernel.Exp}
NMAX = _lib.LML_BATCH_MAX_N


def _prm(k=0, optimize_noise=False, iterations=300, repeats=10, eps_stop=0.0):
    class Prm:
        class kernel:
            noise = 0.01

        class kernel_squared_exp_ard:
            sigma_sq = 1.0

        class opt_rprop:
            pass

        class opt_parallelrepeater:
            epsilon = 1e-2
    Prm.kernel.optimize_noise = optimize_noise
    Prm.kernel_squared_exp_ard.k = k
    Prm.opt_rprop.iterations, Prm.opt_rprop.eps_stop = iterations, eps_stop
    Prm.opt_parallelrepeater.repeats = repeats
    return Prm


def _gp(kid, n, d, p=1, k=0, optimize_noise=False, seed=3, **kw):
    P = _prm(k, optimize_noise, **kw)
    X = synth.points(seed, n, d)
    Y = np.stack([synth.targets(X) * (1 + 0.5 * q) + q for q in range(p)], axis=1)
    gp = model.GP(d, p, params=P, kernel=KERNELS[kid], mean=mean.Data)
    gp.compute(X, Y)
    return gp, P


def _rows(gp, R, seed=0):
    """R h-param vectors around the functor's defaults: long and short length scales, larger and smaller signal variance."""
    k = gp.kernel_function()
    rng = np.random.default_rng(seed)
    H = np.tile(k.h_params(), (R, 1)) + rng.uniform(-1.2, 0.8, (R, k.h_params_size()))
    nk = k.params_size()
    if nk > gp.dim_in() + 1:  # SE-ARD Lambda entries: small
        H[:, gp.dim_in():nk - 1] *= 0.3
    if k.optimize_noise():
        H[:, -1] = rng.uniform(-3.0, -1.0, R)
    return H


def _single(gp, h):
    """today's path: a copy of the GP refitted at h (KernelLFOptimization's evaluation)"""
    g = gp.copy()
    g.kernel_function().set_h_params(h)
    g.recompute(False)
    return g.compute_log_lik(), g.compute_kernel_grad_log_lik(), g.chol_info()


def _close(lik, grad, lik_ref, grad_ref):
    assert abs(lik - lik_ref) <= 1e-11 * max(1.0, abs(lik_ref)), (lik, lik_ref)
    assert np.abs(grad - grad_ref).max() <= 1e-9 * max(1.0, np.abs(grad_ref).max()), (grad, grad_ref)


CASES = [  # kernel id, N, D, P, Lambda k, optimize_noise
    (0, 3, 1, 1, 0, False), (0, 8, 2, 1, 0, False), (1, 60, 3, 1, 0, False), (2, 127, 4, 1, 0, True), (3, 128, 3, 1, 0, False),
    (0, 129, 6, 1, 0, False), (1, 150, 6, 2, 0, False), (0, 190, 2, 1, 2, False), (2, NMAX - 1, 6, 1, 0, False),
    (3, 160, 5, 1, 0, True), (0, NMAX, 6, 1, 0, True), (1, NMAX, 6, 1, 0, False),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "k%d_n%d_d%d_p%d_lam%d_noise%d" % (c[0], c[1], c[2], c[3], c[4], c[5]))
def test_rows_match_single_path(case):
    kid, n, d, p, k, on = case
    gp, _ = _gp(kid, n, d, p, k, on)
    H = _rows(gp, 7, seed=n)
    lik, grad, info = gp.lml_grad_batch(H)
    assert (info == 0).all()
    for r in range(7):
        l1, g1, i1 = _single(gp, H[r])
        assert i1 == 0
        _close(lik[r], grad[r], l1, g1)
    lik2, grad2, _ = gp.lml_grad_batch(H, compute_grad=False)
    assert grad2 is None and np.array_equal(lik2, lik)


@pytest.mark.parametrize("kid", [0, 1, 2, 3])
def test_rows_match_oracle(kid):
    from oracle import oracle as O
    for n in (8, 60, 129):
        gp, _ = _gp(kid, n, 3)
        H = _rows(gp, 5, seed=kid)
        lik, grad, _ = gp.lml_grad_batch(H)
        og = O.OracleGP()
        X = synth.points(3, n, 3)
        og.set_data(X, gp.obs_mean())
        og.set_kernel(kid, H[0], 0.01)
        og.fit()
        for r in range(5):
            lo, go = og.lml_eval(H[r], True)
            _close(lik[r], grad[r], lo, go)


@pytest.mark.parametrize("n", [60, 200])
@pytest.mark.parametrize("R", [1, 7, 133, 1000])
def test_deterministic_across_batches(n, R):
    gp, _ = _gp(0, n, 4, optimize_noise=True)
    H = _rows(gp, R, seed=R)
    lik, grad, info = gp.lml_grad_batch(H)
    assert np.isfinite(lik).all() and (info == 0).all()
    again = gp.lml_grad_batch(H)
    assert np.array_equal(again[0], lik) and np.array_equal(again[1], grad)
    perm = np.random.default_rng(1).permutation(R)
    pl, pg, _ = gp.lml_grad_batch(H[perm])
    assert np.array_equal(pl, lik[perm]) and np.array_equal(pg, grad[perm])
    for r in {0, R // 2, R - 1}:
        al, ag, _ = gp.lml_grad_batch(H[r:r + 1])
        assert al[0] == lik[r] and np.array_equal(ag[0], grad[r])
    for r in range(0, R, max(1, R // 5)):  # a sample of rows against today's path
        l1, g1, _ = _single(gp, H[r])
        _close(lik[r], grad[r], l1, g1)


def _raw_batch(gp, H, noise, optimize_noise=0):
    lib = _lib.load()
    H = np.ascontiguousarray(H, dtype=np.float64)
    noise = np.ascontiguousarray(noise, dtype=np.float64)
    R = H.shape[0]
    nh = H.shape[1] + optimize_noise
    lik, grad, info = np.empty(R), np.empty((R, nh)), np.empty(R, dtype=np.int32)
    rc = lib.lb_lml_grad_batch(gp._h, gp.kernel_function().kernel_id, R, H.shape[1], H.ctypes.data, noise.ctypes.data,
                               optimize_noise, lik.ctypes.data, grad.ctypes.data, info.ctypes.data)
    return rc, lik, grad, info


@pytest.mark.parametrize("n", [40, 150])
def test_non_positive_pivot(n):
    gp, _ = _gp(1, n, 3)
    k = gp.kernel_function()
    H = np.tile(k.params(), (3, 1))
    H[1, 0] = -0.7
    noise = np.array([0.01, -2.0 - 1e-8, 0.02])  # row 1: k(x, x) + noise + 1e-8 = -1 at the first pivot
    rc, lik, grad, info = _raw_batch(gp, H, noise)
    assert rc == 0
    assert info.tolist() == [0, 1, 0]
    assert math.isnan(lik[1]) and np.isnan(grad[1]).all()
    rc0, l0, g0, _ = _raw_batch(gp, H[[0, 2]], noise[[0, 2]])
    assert np.array_equal(l0, lik[[0, 2]]) and np.array_equal(g0, grad[[0, 2]])
    # today's path reports the same pivot, and its likelihood is not finite there
    lib = _lib.load()
    g = gp.copy()
    hp = np.ascontiguousarray(H[1])
    assert lib.lb_set_kernel(g._h, k.kernel_id, hp.ctypes.data, hp.size, C.c_double(noise[1])) == 0
    assert lib.lb_fit(g._h) == info[1]
    out = C.c_double()
    lib.lb_log_lik(g._h, C.addressof(out))
    assert not math.isfinite(out.value)


@pytest.mark.parametrize("n", [40, 150])
def test_non_positive_pivot_inside_the_factor(n):
    """A duplicated sample with a negative noise: the first n - 5 pivots stay near 0.8 (short length scale, K close to
    the identity) and the duplicate's pivot is about -0.45, so both factors must stop at the same index inside the matrix."""
    P = _prm()
    X = synth.points(5, n, 3)
    X[n - 5] = X[7]
    y = synth.targets(X)[:, None]
    gp = model.GP(3, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    gp.compute(X, y)
    H = np.array([[-4.5, 0.0], [-4.5, 0.0], [-0.5, 0.1]])
    noise = np.array([-0.2 - 1e-8, 0.01, 0.01])
    rc, lik, grad, info = _raw_batch(gp, H, noise)
    assert rc == 0 and info.tolist() == [n - 4, 0, 0]
    assert math.isnan(lik[0]) and np.isnan(grad[0]).all() and np.isfinite(lik[1:]).all()
    lib = _lib.load()
    g = gp.copy()
    hp = np.ascontiguousarray(H[0])
    assert lib.lb_set_kernel(g._h, 1, hp.ctypes.data, hp.size, C.c_double(noise[0])) == 0
    assert lib.lb_fit(g._h) == n - 4


def test_model_state_and_launches():
    gp, _ = _gp(0, 200, 6)
    Xq = synth.points(9, 300, 6)
    L0, a0 = gp.matrixL(), gp.alpha()
    mu0, s0 = gp.query_batch(Xq)
    ll0 = gp.compute_log_lik()
    before = gp.launch_count()
    gp.lml_grad_batch(_rows(gp, 40))
    assert gp.launch_count() - before == 1
    before = gp.launch_count()
    gp.lml_grad_batch(_rows(gp, 1000), compute_grad=False)
    assert gp.launch_count() - before == 1
    assert np.array_equal(gp.matrixL(), L0) and np.array_equal(gp.alpha(), a0)
    mu1, s1 = gp.query_batch(Xq)
    assert np.array_equal(mu0, mu1) and np.array_equal(s0, s1)
    assert gp.compute_log_lik() == ll0


def test_error_codes():
    lib = _lib.load()
    gp, _ = _gp(0, 50, 3)
    H = _rows(gp, 2)
    nk = gp.kernel_function().params_size()
    own = np.ascontiguousarray(H[:, :nk])
    noise = np.full(2, 0.01)
    lik, grad, info = np.empty(2), np.empty((2, nk)), np.empty(2, dtype=np.int32)

    def call(h=gp._h, kid=0, R=2, nh=nk, hp=own, no=noise):
        return lib.lb_lml_grad_batch(h, kid, R, nh, hp.ctypes.data, no.ctypes.data, 0, lik.ctypes.data, grad.ctypes.data,
                                     info.ctypes.data)
    assert call() == 0
    assert call(R=0) == -1
    assert call(kid=7) == -1
    assert call(nh=nk + 1) == -1
    bad = own.copy()
    bad[1, 0] = np.nan
    assert call(hp=bad) == -1
    assert call(no=np.array([0.01, np.inf])) == -1
    big = np.zeros(1 + 3 + 3 * 5)  # Lambda k = 5 > 4
    assert lib.lb_lml_grad_batch(gp._h, 0, 1, big.size, big.ctypes.data, noise.ctypes.data, 0, lik.ctypes.data, None, None) == -5
    empty = model.GP(3, 1)
    assert call(h=empty._h) == -3
    large, _ = _gp(1, NMAX + 1, 2)
    hp = np.ascontiguousarray(np.zeros((2, 2)))
    assert lib.lb_lml_grad_batch(large._h, 1, 2, 2, hp.ctypes.data, noise.ctypes.data, 0, lik.ctypes.data, None, None) == -5


def test_dev_variant_matches_host():
    torch = pytest.importorskip("torch")
    lib = _lib.load()
    gp, _ = _gp(2, 100, 3)
    H = np.ascontiguousarray(_rows(gp, 9))
    noise = np.full(9, 0.01)
    lik, grad, _ = gp.lml_grad_batch(H)
    dH, dN = torch.tensor(H, device="cuda"), torch.tensor(noise, device="cuda")
    dL, dG, dI = torch.empty(9, dtype=torch.float64, device="cuda"), torch.empty((9, 2), dtype=torch.float64, device="cuda"), \
        torch.empty(9, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert lib.lb_lml_grad_batch_dev(gp._h, 2, 9, 2, dH.data_ptr(), dN.data_ptr(), 0, dL.data_ptr(), dG.data_ptr(), dI.data_ptr()) == 0
    assert np.array_equal(dL.cpu().numpy(), lik) and np.array_equal(dG.cpu().numpy(), grad)
    assert (dI.cpu().numpy() == 0).all()


def test_concurrent_calls_and_queries():
    gp, _ = _gp(1, 180, 4)
    H = _rows(gp, 20)
    Xq = synth.points(4, 500, 4)
    want_l, want_g, _ = gp.lml_grad_batch(H)
    want_mu, want_s2 = gp.query_batch(Xq)
    errs = []

    def batches():
        try:
            for _ in range(20):
                lik, grad, _ = gp.lml_grad_batch(H)
                assert np.array_equal(lik, want_l) and np.array_equal(grad, want_g)
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    def queries():
        try:
            for _ in range(20):
                mu, s2 = gp.query_batch(Xq)
                assert np.array_equal(mu, want_mu) and np.array_equal(s2, want_s2)
        except Exception as e:  # pragma: no cover
            errs.append(e)
    ts = [threading.Thread(target=batches), threading.Thread(target=queries), threading.Thread(target=batches)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def _fit_both(kid, n, d, iterations, seed=7, **kw):
    out = []
    for batched in (False, True):
        gp, P = _gp(kid, n, d, iterations=iterations, **kw)
        rng = np.random.default_rng(seed)
        rep = opt.BatchedParallelRepeater(P, rng=rng) if batched else opt.ParallelRepeater(P, opt.Rprop(P), rng=rng)
        model.KernelLFOpt(P, rep)(gp)
        out.append((gp.kernel_function().h_params(), gp.get_log_lik()))
    return out


@pytest.mark.parametrize("case", [(0, 60, False), (0, 200, False), (0, 500, False), (1, 120, False), (2, 200, True), (0, 150, True)],
                         ids=lambda c: "k%d_n%d_noise%d" % c)
def test_kernel_lf_opt_batched_matches_sequential(case):
    kid, n, on = case
    (h0, l0), (h1, l1) = _fit_both(kid, n, 3, 30, optimize_noise=on)
    assert np.abs(h1 - h0).max() <= 1e-9
    assert abs(l1 - l0) <= 1e-10 * abs(l0)


def test_full_length_lanes_replay_rprop_on_single_path():
    """300 iterations: every lane's recorded trajectory is a valid Rprop run on today's path's values (the sign pattern of the
    single path's gradient reproduces each step; the path may diverge from the sequential run where a gradient component is
    within rounding of zero, so the trajectory is replayed rather than compared)."""
    gp, P = _gp(1, 200, 4, iterations=300)
    f = model.hp_opt._KernelLFOptimization(gp)
    calls = []

    class Rec:
        def batch(self, X, compute_grad):
            lik, grad = f.batch(X, compute_grad)
            calls.append((X.copy(), lik, grad))
            return lik, grad
    starts = np.tile(gp.kernel_function().h_params(), (3, 1)) + np.random.default_rng(0).uniform(-0.5, 0.5, (3, 2))
    opt.BatchedRprop(P)(Rec(), starts, False)
    assert len(calls) == 300
    for r in range(3):
        traj = np.stack([c[0][r] for c in calls])
        delta, gold = np.full(2, 0.1), np.zeros(2)
        for t in range(len(traj) - 1):
            l1, g1, _ = _single(gp, traj[t])
            g = -np.asarray(g1)
            go = gold * g
            delta = np.where(go > 0, np.minimum(delta * 1.2, 50.0), delta)
            delta = np.where(go < 0, np.maximum(delta * 0.5, 1e-6), delta)
            g = np.where(go < 0, 0.0, g)
            step = traj[t + 1] - traj[t]
            expect = -np.sign(g) * delta
            assert np.allclose(step, expect, rtol=1e-12, atol=1e-15), (r, t)
            gold = g


def test_above_bound_equals_sequential():
    (h0, l0), (h1, l1) = _fit_both(1, NMAX + 8, 2, 4, repeats=3)
    assert np.array_equal(h0, h1) and l0 == l1


def test_boptimizer_loop_with_batched_fit():
    from limbo_b200 import acqui, bayes_opt

    class Prm:
        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 20

        class bayes_opt_boptimizer:
            hp_period = 1

        class opt_rprop:
            iterations = 50
    gp = model.GP(2, 1, params=Prm, kernel=kernel.SquaredExpARD, mean=mean.Data,
                  hp_opt=model.KernelLFOpt(Prm, opt.BatchedParallelRepeater(Prm, rng=np.random.default_rng(0))))
    bo = bayes_opt.BOptimizer(gp, Prm, acqui=acqui.UCB, rng=np.random.default_rng(1))
    bo.optimize(lambda x: np.array([-np.sum((x - 0.3) ** 2)]), 2)
    assert len(bo.samples()) == 30
    assert np.isfinite(gp.get_log_lik())


GOLDEN = sorted(__import__("glob").glob(__import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)),
                                                                  "golden", "lml_batch", "*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[p.split("/")[-1][:-4] for p in GOLDEN])
def test_rows_match_reference_fixtures(path):
    """Every row against the reference's own log-likelihood and gradient (tests/golden/make_golden_lml_batch.py), at the tolerances
    of test_golden.py: lb_lml_grad_batch up to LB_LML_BATCH_MAX_N, the batch objective's row-by-row path above it."""
    g = np.load(path)
    kid, on = int(g["kernel_id"]), bool(g["optimize_noise"])
    P = _prm(2 if kid == 4 else 0, on)
    P.kernel.noise = float(g["noise"])
    X, Y = g["X"], g["Y"]
    gp = model.GP(X.shape[1], Y.shape[1], params=P, kernel=KERNELS[kid % 4], mean=mean.Data)
    gp.compute(X, Y)
    H = g["H"]
    if X.shape[0] <= NMAX:
        lik, grad, info = gp.lml_grad_batch(H)
        assert (info == 0).all()
    else:
        lik, grad = model.hp_opt._KernelLFOptimization(gp).batch(H, True)
    for r in range(H.shape[0]):
        _close(lik[r], grad[r], g["lik"][r], g["grad"][r])


def test_cpp_dropin():
    run_dropin("lml_batch_dropin_test", "LML BATCH DROPIN OK")
