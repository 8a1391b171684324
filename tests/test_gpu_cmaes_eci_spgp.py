"""Batched CMA-ES on the device over ECI (lb_eci_cmaes) and over the pseudo-input sparse GP (lb_spgp_acq_cmaes), with the SPGP
_dev scorers it runs on (lb_spgp_query_dev, lb_spgp_acq_argmax_dev): the instances' state against the NumPy restatement
(oracle/cmaes.py) after every generation, the scored values against the argmax entry points bit for bit, seeds, the ECI cases
of eci_locked, the error codes, the policies and the C++ drop-ins."""
import numpy as np
import pytest

from oracle import cmaes as OC

pytestmark = pytest.mark.gpu

LB_ERR_ARG, LB_ERR_STATE, LB_ERR_UNSUPPORTED = -1, -3, -5


def _params(noise=1e-4):
    class P:
        class kernel:
            pass

        class acqui_ucb:
            alpha = 0.5

        class acqui_ei:
            jitter = 0.0

        class acqui_eci:
            jitter = 0.0
    P.kernel.noise = noise
    return P


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


def _constraint(X):
    """feasible (>= 1) on a band of the box only"""
    return 1.0 + np.cos(4.0 * X[:, 0] + X[:, -1])


def _eci(D, N=120, seed=11, con="gp", precision="fp64", mean=None):
    from limbo_b200 import acqui, kernel, model, synth
    from limbo_b200 import mean as M
    P = _params()
    X = synth.points(seed, N, D)
    obj = model.GP(D, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean or M.Data, precision=precision)
    obj.compute(list(X), list(synth.targets(X)[:, None]))
    c = None
    if con is not None:
        c = model.GP(D, 1, params=P, kernel=kernel.MaternFiveHalves, mean=M.Constant, precision=precision)
        if con == "gp":
            c.compute(list(X), list(_constraint(X)[:, None]))
    return acqui.ECI(obj, c, params=P)


def _spgp(D, N=400, seed=5, f=None, mean=None):
    """an SPGP computed at its starting vector (the optimiser returns its input), on synth.targets or f"""
    from limbo_b200 import model, synth
    from limbo_b200 import mean as M
    X = synth.points(seed, N, D)
    s = model.SPGP(D, 1, params=_params(), mean=mean or M.Data, hp_opt=lambda fun, init, bounded: init,
                   rng=np.random.default_rng(seed))
    s.compute(X, (f or synth.targets)(X)[:, None])
    return s


def _acq(name, D):
    from limbo_b200 import acqui
    if name == "eci":
        return _eci(D)
    s = _spgp(D)
    return acqui.UCB(s, params=_params()) if name == "spgp_ucb" else acqui.EI(s, params=_params())


def _values(acq, X):
    return acq.argmax_batch(X, return_values=True)[2]


@pytest.mark.parametrize("lam", [0, 24])
@pytest.mark.parametrize("R", [1, 8])
@pytest.mark.parametrize("D", [2, 6])
@pytest.mark.parametrize("which", ["eci", "spgp_ucb", "spgp_ei"])
def test_device_state_matches_oracle(capture, which, D, R, lam):
    """m, sigma, A, the best point and value of every instance after every generation, to 1e-9 relative (as for UCB / EI)."""
    acq = _acq(which, D)
    starts = np.random.default_rng(D * 100 + R).random((R, D))
    G, seed = 6, 4321 + D
    bx, bv, n = acq.cmaes_batch(starts, lam=lam, sigma0=0.5, generations=G, tolx=1e-5, seed=seed)
    states, _, _ = _capture(capture, R, lam if lam else OC.default_lambda(D), D)
    s = OC.Search(starts, lam=lam, sigma0=0.5, tolx=1e-5, seed=seed)
    assert n == G * R * s.k.lam and len(states) == G
    for g in range(G):
        s.step(lambda X: _values(acq, X))
        for r in range(R):
            x = states[g][r]
            m, A = x[:D], x[4 * D + D * D:4 * D + 2 * D * D].reshape(D, D)
            w = f"{which} D={D} R={R} lam={lam} g={g} r={r}"
            assert bool(x[-1]) == bool(s.stopped[r]), w
            _close(m, s.m[r], 1e-9, w + " m")
            _close(x[-3], s.sigma[r], 1e-9, w + " sigma")
            _close(A, s.A[r], 1e-9, w + " A")
            _close(x[3 * D:4 * D], s.best_x[r], 1e-9, w + " best_x")
            assert abs(x[-2] - s.best_val[r]) <= 1e-9 * np.max(np.abs(s.best_val)), w + " best_val"
    ox, ov = s.best()
    _close(bx, ox, 1e-9, "best_x")
    _close(bv, ov, 1e-9, "best_val")


def _eci_dev(lib, acq, X):
    """lb_eci_argmax_dev's values at X over the acquisition's pair, with its f_max and the models' constant means"""
    import torch
    from limbo_b200 import _lib
    from limbo_b200.model._calls import constant_mean
    o, c = acq._model, acq._constraint_model
    D = X.shape[1]
    use_con = c is not None and c.nb_samples() > 0
    dX = torch.from_numpy(np.ascontiguousarray(X)).cuda()
    dv = torch.empty(len(X), dtype=torch.float64, device="cuda")
    db = torch.empty(1, dtype=torch.float64, device="cuda")
    di = torch.empty(1, dtype=torch.int64, device="cuda")
    ep = np.array([acq._f_max, acq._jitter()])
    _lib.check(lib.lb_eci_argmax_dev(o._h, None if c is None else c._h, ep.ctypes.data, len(X), dX.data_ptr(), None,
                                     constant_mean(o, D), None, constant_mean(c, D) if use_con else 0.0, dv.data_ptr(), db.data_ptr(),
                                     di.data_ptr()), "lb_eci_argmax_dev")
    _lib.check(lib.lb_sync(o._h), "lb_sync")
    return dv.cpu().numpy()


@pytest.mark.parametrize("case", ["con", "no_con", "empty_con", "fp16x3"])
def test_eci_values_equal_argmax_dev(capture, case):
    """The last generation's values, as the search scored them, equal lb_eci_argmax_dev (and lb_eci_argmax) on the same candidates
    bit for bit: with a constraint model, without one (None), with a constraint without samples (Pf = 1), and with both handles in
    fp16x3, where the search scores the reduced-precision pair."""
    D, R = 6, 7
    acq = _eci(D, N=300, con={"con": "gp", "no_con": None, "empty_con": "empty", "fp16x3": "gp"}[case],
               precision="fp16x3" if case == "fp16x3" else "fp64")
    starts = np.random.default_rng(5).random((R, D))
    bx, bv, n = acq.cmaes_batch(starts, generations=5, tolx=1e-9, seed=9)
    _, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
    assert n == 5 * R * OC.default_lambda(D)
    assert np.array_equal(_eci_dev(capture, acq, cands), vals)
    assert np.array_equal(_values(acq, cands), vals)
    assert np.array_equal(_values(acq, np.tile(bx, (len(cands), 1)))[0], bv)
    if case in ("no_con", "empty_con"):  # Pf = 1: the search scores EI on the objective
        from limbo_b200 import acqui
        ei = acqui.EI(acq._model, params=_params())
        assert np.array_equal(_values(ei, cands), vals)


def test_eci_objective_without_samples(lib):
    """eci.hpp:86: every value is 0, so the search returns the first start, 0 and 0 evaluations, and launches nothing"""
    from limbo_b200 import acqui, kernel, mean, model
    from limbo_b200.model._calls import cmaes
    D = 3
    obj = model.GP(D, 1, params=_params(), kernel=kernel.MaternFiveHalves, mean=mean.Data)
    con = _eci(D)._constraint_model
    starts = np.random.default_rng(1).random((4, D))
    ep = np.array([0.0, 0.0])
    for c in (con, None):
        x, v, n = obj.eci_cmaes_batch(c, 0.0, 0.0, starts, seed=3)
        assert np.array_equal(x, starts[0]) and v == 0.0 and n == 0
        l0, lc = obj.launch_count(), con.launch_count()
        x, v, n = cmaes(lib, "lb_eci_cmaes", D, obj._h, None if c is None else c._h, ep.ctypes.data, 0.0, 0.0, starts, seed=3)
        assert obj.launch_count() == l0 and con.launch_count() == lc
        assert np.array_equal(x, starts[0]) and v == 0.0 and n == 0
    x, v, n = acqui.ECI(obj, con, params=_params()).cmaes_batch(starts)
    assert np.array_equal(x, starts[0]) and v == 0.0 and n == 0


def test_spgp_dev_entry_points_equal_host(lib):
    """lb_spgp_query_dev equals lb_spgp_query, and lb_spgp_acq_argmax_dev equals lb_spgp_acq_argmax, bit for bit, over more than
    one QCHUNK of candidates, with a device mean and with a constant; neither synchronises the host before its results are read"""
    import torch
    from limbo_b200 import _lib, synth
    s = _spgp(4)
    Mq = 9000
    X = synth.points(77, Mq, 4)
    mu, s2 = s.query_batch(X)
    mean = s.mean_function().batch(X, s)[:, 0]
    dX = torch.from_numpy(X).cuda()
    dmu, ds2 = torch.empty(Mq, dtype=torch.float64, device="cuda"), torch.empty(Mq, dtype=torch.float64, device="cuda")
    _lib.check(lib.lb_spgp_query_dev(s._h, Mq, dX.data_ptr(), int(s._optimized), dmu.data_ptr(), ds2.data_ptr()), "lb_spgp_query_dev")
    torch.cuda.synchronize()
    host_mu = np.empty(Mq)
    host_s2 = np.empty(Mq)
    _lib.check(lib.lb_spgp_query(s._h, Mq, X.ctypes.data, int(s._optimized), host_mu.ctypes.data, host_s2.ctypes.data), "lb_spgp_query")
    assert np.array_equal(dmu.cpu().numpy(), host_mu) and np.array_equal(ds2.cpu().numpy(), host_s2)
    assert np.array_equal(host_mu + mean, mu[:, 0]) and np.array_equal(host_s2, s2)
    for acq_id, ap in ((0, [0.5, 0.0]), (1, [float(mu.max()), 0.01])):
        for dmean in (None, torch.from_numpy(np.ascontiguousarray(mean + 0.25)).cuda()):
            mconst = 0.0 if dmean is not None else float(mean[0])
            best, idx, vals = s.acq_argmax_batch(acq_id, ap, X, return_values=True) if dmean is None else (None, None, None)
            if dmean is not None:
                hv, hb, hi = np.empty(Mq), np.empty(1), np.empty(1, dtype=np.int64)
                m = np.ascontiguousarray(mean + 0.25)
                _lib.check(lib.lb_spgp_acq_argmax(s._h, acq_id, np.array(ap).ctypes.data, Mq, X.ctypes.data, int(s._optimized), m.ctypes.data,
                                                  0.0, hv.ctypes.data, hb.ctypes.data, hi.ctypes.data), "lb_spgp_acq_argmax")
                best, idx, vals = hb[0], hi[0], hv
            dv = torch.empty(Mq, dtype=torch.float64, device="cuda")
            db = torch.empty(1, dtype=torch.float64, device="cuda")
            di = torch.empty(1, dtype=torch.int64, device="cuda")
            _lib.check(lib.lb_spgp_acq_argmax_dev(s._h, acq_id, np.array(ap).ctypes.data, Mq, dX.data_ptr(), int(s._optimized),
                                                  None if dmean is None else dmean.data_ptr(), mconst, dv.data_ptr(), db.data_ptr(),
                                                  di.data_ptr()), "lb_spgp_acq_argmax_dev")
            torch.cuda.synchronize()
            assert np.array_equal(dv.cpu().numpy(), vals) and db.item() == best and di.item() == idx


@pytest.mark.parametrize("which", ["spgp_ucb", "spgp_ei"])
def test_spgp_values_equal_argmax_entry_points(capture, which):
    """The last generation's values equal lb_spgp_acq_argmax and lb_spgp_acq_argmax_dev on the captured candidates bit for bit"""
    import torch
    from limbo_b200 import _lib
    D, R = 6, 7
    acq = _acq(which, D)
    starts = np.random.default_rng(5).random((R, D))
    bx, bv, n = acq.cmaes_batch(starts, generations=5, tolx=1e-9, seed=9)
    _, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
    assert n == 5 * R * OC.default_lambda(D)
    assert np.array_equal(_values(acq, cands), vals)
    assert np.array_equal(_values(acq, np.tile(bx, (len(cands), 1)))[0], bv)
    s = acq._model
    ap = np.array([0.5, 0.0]) if which == "spgp_ucb" else np.array([acq._f_max, 0.0])
    dX = torch.from_numpy(np.ascontiguousarray(cands)).cuda()
    dv = torch.empty(len(cands), dtype=torch.float64, device="cuda")
    db = torch.empty(1, dtype=torch.float64, device="cuda")
    di = torch.empty(1, dtype=torch.int64, device="cuda")
    mconst = float(s.mean_function()(cands[0], s)[0])
    _lib.check(capture.lb_spgp_acq_argmax_dev(s._h, 0 if which == "spgp_ucb" else 1, ap.ctypes.data, len(cands), dX.data_ptr(),
                                              int(s._optimized), None, mconst, dv.data_ptr(), db.data_ptr(), di.data_ptr()),
               "lb_spgp_acq_argmax_dev")
    torch.cuda.synchronize()
    assert np.array_equal(dv.cpu().numpy(), vals)


@pytest.mark.parametrize("which", ["eci", "spgp_ucb"])
def test_same_seed_same_bits(capture, which):
    D, R = 6, 16
    acq = _acq(which, D)
    starts = np.random.default_rng(8).random((R, D))
    runs = []
    for _ in range(2):
        bx, bv, n = acq.cmaes_batch(starts, generations=20, tolx=1e-9, seed=77)
        states, cands, vals = _capture(capture, R, OC.default_lambda(D), D)
        runs.append((bx, bv, n, states, cands, vals))
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    acq.cmaes_batch(starts, generations=20, tolx=1e-9, seed=78)
    _, other, _ = _capture(capture, R, OC.default_lambda(D), D)
    assert not np.array_equal(other, runs[0][4])


def test_error_codes(lib):
    from limbo_b200 import _lib, kernel, mean, model
    from limbo_b200.model._calls import cmaes
    D = 3
    acq = _eci(D)
    o, c = acq._model, acq._constraint_model
    starts = np.full((2, D), 0.5)
    ep = np.array([1.0, 0.0])

    def eci(m0, m1, st=starts, **kw):
        return cmaes(lib, "lb_eci_cmaes", D, m0._h, None if m1 is None else m1._h, ep.ctypes.data, 0.0, 0.0, st, **kw)

    def code(fn):
        with pytest.raises(_lib.LimboB200Error) as e:
            fn()
        return e.value.code
    assert code(lambda: eci(o, o)) == LB_ERR_ARG  # the same handle twice
    other = _eci(2)._constraint_model  # a constraint with samples in another input dimension
    assert code(lambda: eci(o, other)) == LB_ERR_ARG
    bad = starts.copy()
    bad[1, 0] = np.inf
    assert code(lambda: eci(o, c, bad)) == LB_ERR_ARG
    assert code(lambda: eci(o, c, lam=257)) == LB_ERR_UNSUPPORTED
    assert code(lambda: acq.cmaes_batch(starts, sigma0=0.0)) == LB_ERR_ARG

    s = _spgp(D)
    from limbo_b200 import acqui
    ucb = acqui.UCB(s, params=_params())
    assert code(lambda: ucb.cmaes_batch(bad)) == LB_ERR_ARG
    assert code(lambda: ucb.cmaes_batch(starts, lam=257)) == LB_ERR_UNSUPPORTED
    assert code(lambda: s.acq_cmaes_batch(2, [0.5, 0.0], starts)) == LB_ERR_ARG  # acq_id outside UCB / EI
    assert code(lambda: s.acq_cmaes_batch(-1, [0.5, 0.0], starts)) == LB_ERR_ARG
    fresh = model.SPGP(D, 1, params=_params(), mean=mean.Data)  # no lb_spgp_compute yet: the C entry, and the Python guard
    assert code(lambda: cmaes(lib, "lb_spgp_acq_cmaes", D, fresh._h, 0, np.array([0.5, 0.0]).ctypes.data, 1, 0.0, starts)) == LB_ERR_STATE
    with pytest.raises(NotImplementedError):
        fresh.acq_cmaes_batch(0, [0.5, 0.0], starts)
    X = np.random.default_rng(0).random((50, D))
    assert lib.lb_spgp_set_data(fresh._h, 50, D, np.ascontiguousarray(X).ctypes.data, np.zeros(50).ctypes.data) == 0
    assert code(lambda: cmaes(lib, "lb_spgp_acq_cmaes", D, fresh._h, 1, np.array([0.5, 0.0]).ctypes.data, 1, 0.0, starts)) == LB_ERR_STATE


def _random_vs_cmaes(acq, D, seed):
    """(best of the random pass and the search, best of BatchedRandomSearch at the same number of evaluations)"""
    from limbo_b200 import bayes_opt
    rng = np.random.default_rng(seed)
    cand = rng.random((2000, D))
    best0, _, vals = acq.argmax_batch(cand, return_values=True)
    starts = bayes_opt._best_distinct(cand, vals, 16)
    _, bv, n = acq.cmaes_batch(starts, sigma0=0.1, generations=40, tolx=1e-9, seed=seed + 1)
    total = 2000 + n

    class P:
        class opt_batchedrandom:
            candidates = total // 3
            refinements = 2
            shrink = 0.1
    x = bayes_opt.BatchedRandomSearch(P, np.random.default_rng(seed))(acq, D)
    return max(bv, best0), _values(acq, x[None])[0]


@pytest.mark.parametrize("which", ["eci", "spgp_ucb", "spgp_ei"])
def test_beats_random_search_at_equal_evaluations(which):
    """ECI on Hartmann6 under a constraint that rules out part of the box (50 samples of each model), and UCB / EI over an SPGP of
    Hartmann6: on three seeds the search's best value (sigma0 = 0.1, the policy's default) exceeds the best value of
    BatchedRandomSearch given the same number of evaluations."""
    from limbo_b200 import acqui, kernel, mean, model, synth
    P = _params()
    if which == "eci":
        X = synth.points(21, 50, 6)
        obj = model.GP(6, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
        obj.compute(X, synth.hartmann6(X)[:, None])
        con = model.GP(6, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Constant)
        con.compute(X, _constraint(X)[:, None])
        acq = acqui.ECI(obj, con, params=P)
    else:
        s = _spgp(6, N=600, f=synth.hartmann6)
        acq = acqui.UCB(s, params=P) if which == "spgp_ucb" else acqui.EI(s, params=P)
    for seed in range(3):
        c, r = _random_vs_cmaes(acq, 6, seed)
        print(which, seed, "cmaes", c, "random", r)
        assert c > r, (which, seed, c, r)


class _Spy:
    """records every cmaes_batch result of the acquisitions a policy builds"""

    def __init__(self, monkeypatch, cls):
        self.results = []
        orig = cls.cmaes_batch

        def spy(acq, starts, **opts):
            r = orig(acq, starts, **opts)
            self.results.append(r)
            return r
        monkeypatch.setattr(cls, "cmaes_batch", spy)


def test_cboptimizer_and_spgp_boptimizer_with_cmaes_policy(monkeypatch):
    """CBOptimizer + BatchedCmaesSearch and BOptimizer(SPGP) + BatchedCmaesSearch: every iteration runs one device search (a spy
    on cmaes_batch sees evaluations > 0, and the SPGP's launch count grows by more than the random pass's)."""
    from limbo_b200 import acqui, bayes_opt, kernel, mean, model, synth

    class P:
        class kernel:
            noise = 1e-6

        class init_randomsampling:
            samples = 10

        class stop_maxiterations:
            iterations = 4

        class opt_batchedcmaes:
            candidates = 2000
            starts = 8
            generations = 20

        class acqui_eci:
            jitter = 0.0
    spy = _Spy(monkeypatch, acqui.ECI)
    rng = np.random.default_rng(0)
    gp = model.GP(6, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Data)
    con = model.GP(6, 1, params=P, kernel=kernel.MaternFiveHalves, mean=mean.Constant)
    bo = bayes_opt.CBOptimizer(gp, con, params=P, acqui_opt=bayes_opt.BatchedCmaesSearch(P, rng), rng=rng)
    bo.optimize(lambda x: np.array([synth.hartmann6(x[None])[0], _constraint(x[None])[0]]), 6, dim_out=1, nb_constraints=1)
    assert len(bo.samples()) == 14 and len(spy.results) == 4 and all(n > 0 for _, _, n in spy.results)

    spy = _Spy(monkeypatch, acqui.UCB)
    s = model.SPGP(3, 1, params=P, mean=mean.Data, hp_opt=lambda f, init, bounded: init, rng=np.random.default_rng(1))
    rng = np.random.default_rng(2)
    launches = []
    orig = bayes_opt.BatchedCmaesSearch.__call__

    def counted(self, acqui_, dim, bounded=True):
        l0 = s.launch_count()
        x = orig(self, acqui_, dim, bounded)
        launches.append(s.launch_count() - l0)
        return x
    monkeypatch.setattr(bayes_opt.BatchedCmaesSearch, "__call__", counted)
    bo = bayes_opt.BOptimizer(s, params=P, acqui_opt=bayes_opt.BatchedCmaesSearch(P, rng), rng=rng)
    bo.optimize(lambda x: synth.targets(x[None])[:1], 3)
    assert len(bo.samples()) == 14 and len(spy.results) == 4 and all(n > 0 for _, _, n in spy.results)
    l0 = s.launch_count()
    acqui.UCB(s, params=P).argmax_batch(np.random.default_rng(0).random((2000, 3)))
    per_pass = s.launch_count() - l0
    assert all(n > 4 * per_pass for n in launches), (launches, per_pass)


def test_input_dependent_mean_falls_back_to_random_pass():
    from limbo_b200 import acqui, bayes_opt, mean

    class P:
        class opt_batchedcmaes:
            candidates = 100
    starts = np.full((1, 2), 0.5)
    e = _eci(2, mean=mean.FunctionARD)
    s = acqui.UCB(_spgp(2, mean=mean.FunctionARD), params=_params())
    for acq in (e, s):
        with pytest.raises(NotImplementedError):
            acq.cmaes_batch(starts)
        x = bayes_opt.BatchedCmaesSearch(P, np.random.default_rng(0))(acq, 2)
        assert x.shape == (2,)


def test_cpp_cmaes_eci_spgp_dropin():
    from dropin import run_dropin
    run_dropin("cmaes_eci_spgp_dropin_test", "CMAES ECI SPGP DROPIN OK")
