"""Batched CMA-ES on the device (lb_acq_cmaes, lb_ehvi_cmaes; limbo_b200/csrc/cmaes.cu) against the NumPy restatement
(oracle/cmaes.py): the instances' state after every generation, the candidates' values against the argmax entry points, the
same bits from the same seed, the best value against a re-score, the search against BatchedRandomSearch at equal evaluations,
the error codes, the evaluation count and short optimisation loops with the new policy."""
import numpy as np
import pytest

from oracle import cmaes as OC
from oracle import ehvi as E2

pytestmark = pytest.mark.gpu

LB_ERR_ARG, LB_ERR_UNSUPPORTED = -1, -5


def _params(noise=1e-4):
    class P:
        class kernel:
            pass

        class acqui_ucb:
            alpha = 0.5
    P.kernel.noise = noise
    return P


def _gp(D, N=120, seed=11, f=None, precision="fp64"):
    from limbo_b200 import kernel, mean, model, synth
    X = synth.points(seed, N, D)
    y = (f or synth.targets)(X)
    gp = model.GP(D, 1, params=_params(), kernel=kernel.MaternFiveHalves, mean=mean.Data, precision=precision)
    gp.compute(list(X), list(y[:, None]))
    return gp


def _acq(name, gp):
    from limbo_b200 import acqui
    return acqui.UCB(gp, params=_params()) if name == "ucb" else acqui.EI(gp, params=_params())


def _values(acq, X):
    return acq.argmax_batch(X, return_values=True)[2]


def _capture(lib, R, lam, D):
    """(states G x R x S, last candidates R lam x D, last values R lam) of the last search on this thread"""
    n = lib.lb_debug_cmaes_trace(None, 0)
    buf = np.empty(n)
    lib.lb_debug_cmaes_trace(buf.ctypes.data, n)
    S = 4 * D + 2 * D * D + 3
    M = R * lam
    G = (n - M * D - M) // (R * S)
    return buf[:G * R * S].reshape(G, R, S), buf[G * R * S:G * R * S + M * D].reshape(M, D), buf[G * R * S + M * D:]


def _close(a, b, rel, what):
    scale = max(float(np.max(np.abs(b))), 1e-300)
    err = float(np.max(np.abs(np.asarray(a) - np.asarray(b))))
    assert err <= rel * scale, f"{what}: {err} > {rel} * {scale}"


@pytest.fixture
def capture(lib):
    lib.lb_debug_cmaes_capture(1)
    yield lib
    lib.lb_debug_cmaes_capture(0)


@pytest.mark.parametrize("lam", [0, 256])
@pytest.mark.parametrize("R", [1, 7, 64])
@pytest.mark.parametrize("D", [1, 2, 6, 12, 64])
@pytest.mark.parametrize("acq_name", ["ucb", "ei"])
def test_device_state_matches_oracle(capture, acq_name, D, R, lam):
    """m, sigma, A, the best point and value of every instance after every generation, to 1e-9 relative.  The parity run stops
    after a few generations: near convergence the values tie to rounding and the two sides may rank them differently."""
    gp = _gp(D)
    acq = _acq(acq_name, gp)
    rng = np.random.default_rng(D * 100 + R)
    starts = rng.random((R, D))
    G, seed = 6, 1234 + D
    bx, bv, n = acq.cmaes_batch(starts, lam=lam, sigma0=0.5, generations=G, tolx=1e-5, seed=seed)
    states, _, _ = _capture(capture, R, lam if lam else OC.default_lambda(D), D)
    s = OC.Search(starts, lam=lam, sigma0=0.5, tolx=1e-5, seed=seed)
    assert n == G * R * s.k.lam and len(states) == G
    for g in range(G):
        s.step(lambda X: _values(acq, X))
        st = states[g]
        for r in range(R):
            x = st[r]
            m, A = x[:D], x[4 * D + D * D:4 * D + 2 * D * D].reshape(D, D)
            sig, best_val, stop = x[-3], x[-2], x[-1]
            w = f"{acq_name} D={D} R={R} lam={lam} g={g} r={r}"
            assert bool(stop) == bool(s.stopped[r]), w
            _close(m, s.m[r], 1e-9, w + " m")
            _close(sig, s.sigma[r], 1e-9, w + " sigma")
            _close(A, s.A[r], 1e-9, w + " A")
            _close(x[3 * D:4 * D], s.best_x[r], 1e-9, w + " best_x")
            # relative to the largest best value of the generation: EI's far tail (values ~1e-250) amplifies the candidates'
            # last-bit differences far beyond 1e-9 of the value itself
            assert abs(best_val - s.best_val[r]) <= 1e-9 * np.max(np.abs(s.best_val)), w + " best_val"
    ox, ov = s.best()
    _close(bx, ox, 1e-9, "best_x")
    _close(bv, ov, 1e-9, "best_val")


def _dtlz2(x):
    x = np.atleast_2d(x)
    g = ((x[:, 2:] - 0.5) ** 2).sum(axis=1)
    a, b = x[:, 0] * np.pi / 2, x[:, 1] * np.pi / 2
    return -np.stack([(1 + g) * np.cos(a) * np.cos(b), (1 + g) * np.cos(a) * np.sin(b), (1 + g) * np.sin(a)], axis=1)


def _ehvi(K, N=60, D=6, seed=3):
    from limbo_b200 import acqui, kernel, mean, model
    rng = np.random.default_rng(seed)
    X = rng.random((N, D))
    Y = _dtlz2(X)[:, :K]
    ms = []
    for j in range(K):
        m = model.GP(D, 1, params=_params(1e-4), kernel=kernel.MaternFiveHalves, mean=mean.Data)
        m.compute(X, Y[:, j:j + 1])
        ms.append(m)
    return acqui.EHVI(ms, Y[E2.pareto_set(Y)], (-11.0,) * K)


@pytest.mark.parametrize("which", ["ucb", "ei", "ehvi2", "ehvi3"])
def test_candidate_values_equal_argmax_entry_points(capture, which):
    """The last generation's values, as the search scored them, equal lb_acq_argmax / lb_ehvi_argmax / lb_ehvi3d_argmax on the same
    candidates bit for bit; best_val equals a re-score of best_x."""
    D, R = 6, 7
    acq = _acq(which, _gp(D)) if which in ("ucb", "ei") else _ehvi(int(which[-1]), D=D)
    starts = np.random.default_rng(5).random((R, D))
    bx, bv, n = acq.cmaes_batch(starts, generations=5, tolx=1e-9, seed=9)
    _, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
    assert np.array_equal(_values(acq, cands), vals)
    assert np.array_equal(_values(acq, np.tile(bx, (len(cands), 1)))[0], bv)
    assert abs(_values(acq, bx[None])[0] - bv) <= 1e-12 * max(abs(bv), 1e-300)
    assert n == 5 * R * OC.default_lambda(D)


@pytest.mark.parametrize("which", ["ucb", "ehvi3"])
def test_same_seed_same_bits(capture, which):
    D, R = 6, 16
    acq = _acq(which, _gp(D)) if which == "ucb" else _ehvi(3, D=D)
    starts = np.random.default_rng(8).random((R, D))
    runs = []
    for _ in range(2):
        bx, bv, n = acq.cmaes_batch(starts, generations=20, tolx=1e-9, seed=77)
        states, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
        runs.append((bx, bv, n, states, cands, vals))
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    other = acq.cmaes_batch(starts, generations=20, tolx=1e-9, seed=78)
    assert not np.array_equal(other[0], runs[0][0])


def test_evaluation_count_with_early_stop(lib):
    """Every instance stops (tolx) long before `generations`; the host sees it after the next multiple of 8 generations, and
    n_evals counts the candidates scored up to there, as oracle.cmaes.run does."""
    D, R = 2, 4
    acq = _acq("ucb", _gp(D))
    starts = np.random.default_rng(2).random((R, D))
    bx, bv, n = acq.cmaes_batch(starts, generations=500, tolx=1e-3, seed=4)
    ox, ov, on = OC.run(lambda X: _values(acq, X), starts, 500, tolx=1e-3, seed=4)
    lam = OC.default_lambda(D)
    assert n == on and n % (8 * R * lam) == 0 and n < 500 * R * lam
    _close(bx, ox, 1e-6, "best_x")


def test_beats_random_search_at_equal_evaluations():
    """UCB on Hartmann6 and three-objective EHVI on DTLZ2 (D = 6): on fixed seeds, the best value the search finds exceeds the
    best value of BatchedRandomSearch given the same number of evaluations."""
    from limbo_b200 import bayes_opt
    from limbo_b200 import synth
    for acq in (_acq("ucb", _gp(6, N=200, f=synth.hartmann6)), _ehvi(3, N=80, D=6)):
        rng = np.random.default_rng(0)
        cand = rng.random((2000, 6))
        best0, _, vals = acq.argmax_batch(cand, return_values=True)
        starts = bayes_opt._best_distinct(cand, vals, 16)
        _, bv, n = acq.cmaes_batch(starts, generations=40, tolx=1e-9, seed=1)
        total = 2000 + n

        class P:
            class opt_batchedrandom:
                candidates = total // 3
                refinements = 2
                shrink = 0.1
        x = bayes_opt.BatchedRandomSearch(P, np.random.default_rng(0))(acq, 6)
        br = _values(acq, x[None])[0]
        print(type(acq).__name__, "cmaes", max(bv, best0), "random", br, "evaluations", total)
        assert max(bv, best0) > br


def test_reduced_precision_search(capture):
    """lb_acq_cmaes on an fp16x3 handle: the search runs on the reduced-precision scorer, its last generation's values equal
    lb_acq_argmax's on the same candidates and the best value is a value it scored."""
    D, R = 6, 8
    acq = _acq("ucb", _gp(D, N=300, precision="fp16x3"))
    starts = np.random.default_rng(3).random((R, D))
    bx, bv, n = acq.cmaes_batch(starts, generations=10, tolx=1e-9, seed=5)
    _, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
    assert np.array_equal(_values(acq, cands), vals)
    assert np.array_equal(_values(acq, np.tile(bx, (len(cands), 1)))[0], bv)
    assert n == 10 * R * OC.default_lambda(D)


def test_cpp_cmaes_dropin():
    from dropin import run_dropin
    run_dropin("cmaes_dropin_test", "CMAES DROPIN OK")


def test_error_codes(lib):
    """Every LB_ERR_ARG case and lambda > 256.  D > 64 (the other LB_ERR_UNSUPPORTED case) cannot reach the search through a
    handle: lb_set_data already rejects D > 64."""
    from limbo_b200 import _lib
    gp = _acq("ucb", _gp(3))
    starts = np.full((2, 3), 0.5)
    for kw in (dict(sigma0=0.0), dict(sigma0=-1.0), dict(tolx=0.0), dict(tolx=-1.0), dict(generations=0)):
        with pytest.raises(_lib.LimboB200Error) as e:
            gp.cmaes_batch(starts, **kw)
        assert e.value.code == LB_ERR_ARG, kw
    bad = starts.copy()
    bad[1, 2] = np.nan
    with pytest.raises(_lib.LimboB200Error) as e:
        gp.cmaes_batch(bad)
    assert e.value.code == LB_ERR_ARG
    with pytest.raises(_lib.LimboB200Error) as e:
        gp.cmaes_batch(starts[:0])
    assert e.value.code == LB_ERR_ARG
    with pytest.raises(_lib.LimboB200Error) as e:
        gp.cmaes_batch(starts, lam=257)
    assert e.value.code == LB_ERR_UNSUPPORTED
    # the EHVI entry: lb_ehvi_argmax's rules (the same handle twice, a non-finite front)
    eh = _ehvi(2, D=3)
    m0, m1 = eh._models
    with pytest.raises(_lib.LimboB200Error) as e:
        m0.ehvi_cmaes_batch([m0], (-11.0, -11.0), eh._pop, starts)
    assert e.value.code == LB_ERR_ARG
    front = eh._pop.copy()
    front[0, 0] = np.inf
    with pytest.raises(_lib.LimboB200Error) as e:
        m0.ehvi_cmaes_batch([m1], (-11.0, -11.0), front, starts)
    assert e.value.code == LB_ERR_ARG


def test_input_dependent_mean_falls_back_to_random_pass():
    from limbo_b200 import bayes_opt, kernel, mean, model, synth
    X = synth.points(3, 40, 2)
    gp = model.GP(2, 1, params=_params(), kernel=kernel.MaternFiveHalves, mean=mean.FunctionARD)
    gp.compute(X, synth.targets(X)[:, None])
    with pytest.raises(NotImplementedError):
        _acq("ucb", gp).cmaes_batch(np.full((1, 2), 0.5))

    class P:
        class opt_batchedcmaes:
            candidates = 100
    x = bayes_opt.BatchedCmaesSearch(P, np.random.default_rng(0))(_acq("ucb", gp), 2)
    assert x.shape == (2,)


def test_boptimizer_and_three_objective_ehvi_with_cmaes_policy():
    from limbo_b200 import bayes_opt, kernel, mean, model, synth
    from oracle import ehvi3d as E

    class P:
        class kernel:
            noise = 1e-6

        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 6

        class opt_batchedcmaes:
            candidates = 2000
            starts = 8
            generations = 20
    rng = np.random.default_rng(0)
    gp = model.GP(6, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    bo = bayes_opt.BOptimizer(gp, params=P, acqui_opt=bayes_opt.BatchedCmaesSearch(P, rng), rng=rng)
    bo.optimize(lambda x: synth.hartmann6(x[None])[:1], 6)
    assert len(bo.samples()) == 16 and all(np.all((s >= 0) & (s <= 1)) for s in bo.samples())

    r = (-11.0, -11.0, -11.0)
    rng = np.random.default_rng(1)
    be = bayes_opt.Ehvi(params=P, acqui_opt=bayes_opt.BatchedCmaesSearch(P, rng), rng=rng)
    be.optimize(lambda x: _dtlz2(x)[0], 4)
    Y = np.stack(be.observations())
    assert Y.shape == (16, 3)
    assert E.hypervolume3d(Y[E2.pareto_set(Y)], r) > E.hypervolume3d(Y[:10][E2.pareto_set(Y[:10])], r)
